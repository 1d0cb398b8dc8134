"""Thin object wrapper over the ``drl_apex_replay_*`` C-ABI (include/drl_b200.h): the Ape-X prioritized replay memory on
the device.

``buffer_queue.Memory`` (distributed_queue/buffer_queue.py:371-415) keeps its sum tree in ``drl_per_*`` on the host and
its transitions in a Python object array; the learner loop of ``train_apex.py:82-155`` then stacks every minibatch on
the host and copies it to the GPU.  ``NativeApexReplay`` keeps both on the GPU beside a ``NativeApexLearner``: ingest
with the learner's own |td|, stratified sampling, the minibatch gather into a staging slot and the priority update
from the step's |td| run as kernels on the learner's compute stream.  The host draws the uniforms (the reference's
``random.random()``) and keeps the control flow.  Same constants and arithmetic as ``Memory``: for the same uniforms
it samples the same indices (DESIGN.md section 10).
"""
import ctypes as C

import numpy as np

from . import _native as N


class NativeApexReplay:

    def __init__(self, capacity, device=0, input_shape=(84, 84, 4)):
        self.capacity, self.device = int(capacity), int(device)
        self.input_shape = tuple(int(x) for x in input_shape)
        self._h = C.c_void_p()
        N.check(N.lib.drl_apex_replay_create(self.device, self.capacity, C.byref(self._h)))
        self._n_last = 0            # draws of the most recent sample / step

    # ---- lifetime ----------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            N.lib.drl_apex_replay_destroy(self._h)
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
        N.check(N.lib.drl_apex_replay_size(self._h, C.byref(v)))
        return int(v.value)

    @property
    def beta(self):
        v = C.c_double()
        N.check(N.lib.drl_apex_replay_beta(self._h, C.byref(v)))
        return float(v.value)

    def total(self):
        v = C.c_double()
        N.check(N.lib.drl_apex_replay_total(self._h, C.byref(v)))
        return float(v.value)

    # ---- data path ---------------------------------------------------------------
    def add(self, learner, state, next_state, previous_action, action, reward, done, error=None):
        """Memory.add of n transitions in order.  error=None: the priorities are ``learner``'s |td| of these transitions,
        computed on the device (n <= learner.B); otherwise ``error`` [n] (learner may be None)."""
        n = int(np.asarray(state).shape[0])
        arrs = (N.as_c(state, np.uint8, (n,) + self.input_shape, "state"),
                N.as_c(next_state, np.uint8, (n,) + self.input_shape, "next_state"),
                N.as_c(previous_action, np.int32, (n,), "previous_action"),
                N.as_c(action, np.int32, (n,), "action"),
                N.as_c(reward, np.float32, (n,), "reward"),
                N.as_c(N.as_u8(done), np.uint8, (n,), "done"))
        err = None if error is None else N.as_c(error, np.float64, (n,), "error")
        N.check(N.lib.drl_apex_replay_add(self._h, learner._h if learner is not None else None, n,
                                          *[N.ptr(a) for a in arrs], N.ptr(err) if err is not None else None))

    def add_from_queue(self, learner, queue, timeout_ms=-1):
        """``add`` of the oldest record of an ``ApexDeviceFIFOQueue`` with ``learner``'s |td| as the priorities, read
        straight from the queue's GPU memory (queue.trajectory <= learner.B).  Blocks while the queue is empty;
        ``timeout_ms`` >= 0 raises ``TimeoutError_`` with nothing changed."""
        from .distributed_queue.buffer_queue import ApexDeviceFIFOQueue
        if not isinstance(queue, ApexDeviceFIFOQueue):
            raise TypeError("add_from_queue: queue must be an ApexDeviceFIFOQueue, got %s" % type(queue).__name__)
        N.check(N.lib.drl_apex_replay_add_from_queue(self._h, learner._h, queue._q, int(timeout_ms)))

    def step_async(self, learner, slot, u01):
        """Sample learner.B draws with the uniforms ``u01`` -> gather into ``slot`` -> learner step -> priority update.
        ``learner.wait()`` returns (scalars, td_error) afterwards."""
        u = N.as_c(u01, np.float64, (learner.B,), "u01")
        N.check(N.lib.drl_apex_replay_step_async(self._h, learner._h, int(slot), N.ptr(u)))
        self._n_last = learner.B

    def sample(self, n, u01):
        """Memory.sample's draws -> (tree_index, data_index, priority, is_weight), each [n]."""
        u = N.as_c(u01, np.float64, (n,), "u01")
        ti, di = np.empty(n, np.int64), np.empty(n, np.int64)
        pr, w = np.empty(n, np.float64), np.empty(n, np.float64)
        N.check(N.lib.drl_apex_replay_sample(self._h, n, N.ptr(u), N.ptr(ti), N.ptr(di), N.ptr(pr), N.ptr(w)))
        self._n_last = n
        return ti, di, pr, w

    def update(self, idx, err):
        """Memory.update for each (idx[i], err[i]) in order."""
        ti = N.as_c(idx, np.int64, None, "idx").reshape(-1)
        e = N.as_c(err, np.float64, (ti.size,), "err")
        N.check(N.lib.drl_apex_replay_update(self._h, ti.size, N.ptr(ti), N.ptr(e)))

    def last_sample(self):
        """The draws of the most recent sample or step: (tree_index, priority, is_weight)."""
        n = self._n_last
        ti, pr, w = np.empty(n, np.int64), np.empty(n, np.float64), np.empty(n, np.float64)
        N.check(N.lib.drl_apex_replay_last_sample(self._h, N.ptr(ti), N.ptr(pr), N.ptr(w)))
        return ti, pr, w

    def read(self, data_index, n=1):
        """Rows [data_index, data_index + n) of the storage as a dict of arrays."""
        n = int(n)
        out = dict(state=np.empty((n,) + self.input_shape, np.uint8),
                   next_state=np.empty((n,) + self.input_shape, np.uint8),
                   previous_action=np.empty(n, np.int32), action=np.empty(n, np.int32),
                   reward=np.empty(n, np.float32), done=np.empty(n, np.uint8))
        N.check(N.lib.drl_apex_replay_read(self._h, int(data_index), n,
                                           *[N.ptr(out[k]) for k in ("state", "next_state", "previous_action",
                                                                     "action", "reward", "done")]))
        return out
