"""Thin object wrapper over the ``drl_r2d2_replay_*`` C-ABI (include/drl_b200.h): the R2D2 prioritized sequence replay
memory on the device.

The learner loop of ``train_r2d2.py:87-165`` computes every queued sequence's priority with its own ``get_td_error``
call, keeps the sequences in ``buffer_queue.Memory``'s Python object array, and for every step builds seven lists,
stacks them on the host and copies the minibatch to the GPU.  ``NativeR2D2Replay`` keeps the sequences and the sum tree
on the GPU beside a ``NativeR2D2Learner``: ingest with the learner's |td| of a whole batch of sequences, stratified
sampling, the minibatch gather into a staging slot and the priority update from the step's |td| run as kernels on the
learner's compute stream.  The host draws the uniforms (the reference's ``random.random()``) and keeps the control
flow.  Same constants and arithmetic as ``Memory``: for the same uniforms it samples the same indices (DESIGN.md
section 11).  A record keeps step 0 of the stored (h, c), the only step the learner reads, as ``lstm_size`` floats each
(64, 256 or 512: the width of the learners it serves).
"""
import ctypes as C

import numpy as np

from . import _native as N

class NativeR2D2Replay:

    def __init__(self, capacity, seq_len=15, num_action=4, input_shape=(84, 84, 1), device=0, lstm_size=64):
        self.capacity, self.device = int(capacity), int(device)
        self.S, self.A, self.L = int(seq_len), int(num_action), int(lstm_size)
        self.input_shape = tuple(int(x) for x in input_shape)
        self._h = C.c_void_p()
        N.check(N.lib.drl_r2d2_replay_create_lstm(self.device, self.capacity, self.S, self.input_shape[-1], self.A,
                                                  self.L, C.byref(self._h)))
        self._n_last = 0            # draws of the most recent sample / step

    # ---- lifetime ----------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            N.lib.drl_r2d2_replay_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- state -------------------------------------------------------------------
    @property
    def n_entries(self):
        v = C.c_int64()
        N.check(N.lib.drl_r2d2_replay_size(self._h, C.byref(v)))
        return int(v.value)

    @property
    def beta(self):
        v = C.c_double()
        N.check(N.lib.drl_r2d2_replay_beta(self._h, C.byref(v)))
        return float(v.value)

    def total(self):
        v = C.c_double()
        N.check(N.lib.drl_r2d2_replay_total(self._h, C.byref(v)))
        return float(v.value)

    # ---- data path ---------------------------------------------------------------
    def add(self, learner, state, previous_action, action, h0, c0, reward, done, error=None):
        """Memory.add of n sequences in order: state [n, S, H, W, C], previous_action / action / reward / done [n, S],
        h0 / c0 [n, lstm_size] (step 0 of the stored states).  error=None: the priorities are ``learner``'s |td| of these
        sequences, computed on the device (n <= learner.B); otherwise ``error`` [n] (learner may be None)."""
        n, S = int(np.asarray(state).shape[0]), self.S
        arrs = (N.as_c(state, np.uint8, (n, S) + self.input_shape, "state"),
                N.as_c(previous_action, np.int32, (n, S), "previous_action"),
                N.as_c(action, np.int32, (n, S), "action"),
                N.as_c(h0, np.float32, (n, self.L), "h0"), N.as_c(c0, np.float32, (n, self.L), "c0"),
                N.as_c(reward, np.float32, (n, S), "reward"),
                N.as_c(N.as_u8(done), np.uint8, (n, S), "done"))
        err = None if error is None else N.as_c(error, np.float64, (n,), "error")
        N.check(N.lib.drl_r2d2_replay_add(self._h, learner._h if learner is not None else None, n,
                                          *[N.ptr(a) for a in arrs], N.ptr(err) if err is not None else None))

    def add_from_queue(self, learner, queue, timeout_ms=-1):
        """``add`` of the oldest full batch of an ``R2D2DeviceFIFOQueue`` with ``learner``'s |td| as the priorities,
        read straight from the queue's GPU memory (queue.batch_size <= learner.B).  Blocks while fewer than a batch
        of sequences are queued; ``timeout_ms`` >= 0 raises ``TimeoutError_`` with nothing changed."""
        from .distributed_queue.buffer_queue import R2D2DeviceFIFOQueue
        if not isinstance(queue, R2D2DeviceFIFOQueue):
            raise TypeError("add_from_queue: queue must be an R2D2DeviceFIFOQueue, got %s" % type(queue).__name__)
        N.check(N.lib.drl_r2d2_replay_add_from_queue(self._h, learner._h, queue._q, int(timeout_ms)))

    def step_async(self, learner, slot, u01):
        """Sample learner.B draws with the uniforms ``u01`` -> gather into ``slot`` -> learner step -> priority update.
        ``learner.wait()`` returns (scalars, td_error) afterwards."""
        u = N.as_c(u01, np.float64, (learner.B,), "u01")
        N.check(N.lib.drl_r2d2_replay_step_async(self._h, learner._h, int(slot), N.ptr(u)))
        self._n_last = learner.B

    def sample(self, n, u01):
        """Memory.sample's draws -> (tree_index, data_index, priority, is_weight), each [n]."""
        u = N.as_c(u01, np.float64, (n,), "u01")
        ti, di = np.empty(n, np.int64), np.empty(n, np.int64)
        pr, w = np.empty(n, np.float64), np.empty(n, np.float64)
        N.check(N.lib.drl_r2d2_replay_sample(self._h, n, N.ptr(u), N.ptr(ti), N.ptr(di), N.ptr(pr), N.ptr(w)))
        self._n_last = n
        return ti, di, pr, w

    def update(self, idx, err):
        """Memory.update for each (idx[i], err[i]) in order."""
        ti = N.as_c(idx, np.int64, None, "idx").reshape(-1)
        e = N.as_c(err, np.float64, (ti.size,), "err")
        N.check(N.lib.drl_r2d2_replay_update(self._h, ti.size, N.ptr(ti), N.ptr(e)))

    def last_sample(self):
        """The draws of the most recent sample or step: (tree_index, priority, is_weight)."""
        n = self._n_last
        ti, pr, w = np.empty(n, np.int64), np.empty(n, np.float64), np.empty(n, np.float64)
        N.check(N.lib.drl_r2d2_replay_last_sample(self._h, N.ptr(ti), N.ptr(pr), N.ptr(w)))
        return ti, pr, w

    def read(self, data_index, n=1):
        """Rows [data_index, data_index + n) of the storage as a dict of arrays (h0 / c0 [n, lstm_size])."""
        n, S = int(n), self.S
        out = dict(state=np.empty((n, S) + self.input_shape, np.uint8),
                   previous_action=np.empty((n, S), np.int32), action=np.empty((n, S), np.int32),
                   h0=np.empty((n, self.L), np.float32), c0=np.empty((n, self.L), np.float32),
                   reward=np.empty((n, S), np.float32), done=np.empty((n, S), np.uint8))
        N.check(N.lib.drl_r2d2_replay_read(self._h, int(data_index), n,
                                           *[N.ptr(out[k]) for k in ("state", "previous_action", "action", "h0", "c0",
                                                                     "reward", "done")]))
        return out
