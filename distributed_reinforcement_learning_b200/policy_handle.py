"""The part of the IMPALA, R2D2 and Ape-X / A3C policy-engine wrappers that is the same for all three: each drives one
``drl_<prefix>_*`` policy handle of the C-ABI (include/drl_b200.h), and these entry points differ only in that
prefix.  ``RecorderHandle`` is the same for the recorders of the IMPALA, R2D2 and A3C engines
(``drl_<prefix>_recorder_*``)."""
import ctypes as C

import numpy as np

from . import _native as N

MAX_BATCH = 64


def explore_actions(epsilon, n, num_action):
    """The epsilon-greedy draws of agent/r2d2.py:181-184 for n rows, in row order: ``np.random.rand() > epsilon`` keeps
    the greedy action (-1 here), otherwise ``np.random.choice(num_action)`` is the action.  ``epsilon`` is a scalar or
    one value per row."""
    eps = np.broadcast_to(np.asarray(epsilon, np.float64), (n,))
    out = np.full(n, -1, np.int32)
    for r in range(n):
        if not np.random.rand() > eps[r]:
            out[r] = np.random.choice(num_action)
    return out


class PolicyHandle:
    prefix = None      # "policy", "r2d2_policy" or "apex_policy": the C-ABI prefix

    def _fn(self, name):
        return getattr(N.lib, "drl_%s_%s" % (self.prefix, name))

    def _create(self, cfg):
        self._h = C.c_void_p()
        N.check(self._fn("create")(C.byref(cfg), C.byref(self._h)))
        n = C.c_int64()
        N.check(self._fn("param_count")(self._h, C.byref(n)))
        self.param_count = int(n.value)

    # ---- lifetime ----------------------------------------------------------------
    def close(self):
        # recorders first: a recorder's handle refers to this engine (the garbage collector may finalize the two in
        # either order, so the engine owns the recorders' handle boxes, not the recorders)
        for prefix, r in getattr(self, "_recorder_handles", ()):
            _destroy_recorder(prefix, r)
        self._recorder_handles = []
        if getattr(self, "_h", None) is not None and self._h.value:
            self._fn("destroy")(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- parameters ------------------------------------------------------------------
    def set_params(self, flat):
        """Flat float32 vector of one network in the learner's TF order (the learner's get_params of its main
        network)."""
        a = N.as_c(flat, np.float32, (self.param_count,), "params")
        N.check(self._fn("set_params")(self._h, N.ptr(a), a.size))

    def get_params(self):
        a = np.empty(self.param_count, np.float32)
        N.check(self._fn("get_params")(self._h, N.ptr(a), a.size))
        return a

    def _learner_type(self):
        raise NotImplementedError

    def sync_from(self, learner):
        """parameter_sync from a learner of this family on the same device: device-to-device copy of its main
        parameters after all work enqueued on it so far (a step in flight included); the learner's next update waits
        for the copy."""
        cls = self._learner_type()
        if not isinstance(learner, cls):
            raise TypeError("sync_from takes a %s, got %s" % (cls.__name__, type(learner).__name__))
        N.check(self._fn("sync_from_learner")(self._h, learner._h))

    def last_act_ms(self):
        """Device time of the last act (input copy + kernels), from CUDA events on the policy's stream."""
        ms = C.c_float()
        N.check(self._fn("last_act_ms")(self._h, C.byref(ms)))
        return float(ms.value)

    # ---- test aids -------------------------------------------------------------------
    def buffer_dims(self):
        """(n, splits, N): the rows of the most recent act (0 before the first) and the split count and columns of its
        "zpart" buffer."""
        out = (C.c_int32 * 3)()
        N.check(self._fn("buffer_dims")(self._h, out))
        return int(out[0]), int(out[1]), int(out[2])

    def read_buffer(self, name):
        """A float32 copy of one buffer of the most recent act (n rows), in device layout: "a1" [n, 20, 20, 32], "a2"
        [n, 9, 9, 64], "a3" [n, 3136], "e1" / "table" [A, 256], "zpart" [splits, n, N] (the first skinny GEMM's
        partial sums per K split)."""
        n, splits, cols = self.buffer_dims()
        shape = {"a1": (n, 20, 20, 32), "a2": (n, 9, 9, 64), "a3": (n, 3136), "e1": (self.A, 256),
                 "table": (self.A, 256), "zpart": (splits, n, cols)}.get(name, (0,))
        a = np.empty(int(np.prod(shape)), np.float32)
        N.check(self._fn("read_buffer")(self._h, name.encode(), N.ptr(a), a.size))
        return a.reshape(shape)

    # ---- inputs ----------------------------------------------------------------------
    def _inputs(self, state, previous_action):
        """-> n, state uint8 [n] + input_shape, previous_action int32 [n] in [0, A), as C-contiguous arrays."""
        st = np.asarray(state)
        if st.dtype != np.uint8:
            raise ValueError("state: expected uint8 frames, got %s" % st.dtype)
        if st.ndim != 4:
            raise ValueError("state: expected shape (n,) + %s, got %s" % (self.input_shape, st.shape))
        n = st.shape[0]
        if not 1 <= n <= self.max_batch:
            raise ValueError("state: n = %d rows, this policy serves 1..%d" % (n, self.max_batch))
        st = N.as_c(st, np.uint8, (n,) + self.input_shape, "state")
        pa_in = np.asarray(previous_action)
        if not np.issubdtype(pa_in.dtype, np.integer):
            raise ValueError("previous_action: expected integers, got %s" % pa_in.dtype)
        pa = N.as_c(pa_in, np.int32, (n,), "previous_action")
        if pa.min() < 0 or pa.max() >= self.A:
            raise ValueError("previous_action: values must lie in [0, %d)" % self.A)
        return n, st, pa

    def _explore(self, n, epsilon, explore_action):
        """The explore actions of n rows (int32 [n], -1 = greedy) from ``epsilon`` (drawn by ``explore_actions``) or
        ``explore_action``; None when neither is given (every row greedy)."""
        if epsilon is not None and explore_action is not None:
            raise ValueError("pass epsilon or explore_action, not both")
        if epsilon is not None:
            explore_action = explore_actions(epsilon, n, self.A)
        if explore_action is None:
            return None
        ex_in = np.asarray(explore_action)
        if not np.issubdtype(ex_in.dtype, np.integer):
            raise ValueError("explore_action: expected integers, got %s" % ex_in.dtype)
        ex = N.as_c(ex_in, np.int32, (n,), "explore_action")
        if ex.min() < -1 or ex.max() >= self.A:
            raise ValueError("explore_action: values must lie in [-1, %d)" % self.A)
        return ex


def _destroy_recorder(prefix, handle):
    if handle.value:
        getattr(N.lib, "drl_%s_recorder_destroy" % prefix)(handle)
        handle.value = None


class RecorderHandle:
    """A ``drl_<prefix>_recorder_*`` handle that binds one policy engine to one device queue for n rows.  The family's
    class binds it (``_bind``) and implements ``act``."""
    prefix = None      # the C-ABI prefix of the recorder's entry points; None: the policy's

    def _prefix(self):
        return self.prefix or self.policy.prefix

    def _bind(self, policy, queue, queue_type, n, T):
        """queue must be a ``queue_type``; T: its steps per record."""
        if not isinstance(queue, queue_type):
            raise TypeError("recorder: queue must be a %s, got %s" % (queue_type.__name__, type(queue).__name__))
        n = int(n)
        if not 1 <= n <= policy.max_batch:
            raise ValueError("recorder: n = %d rows, the policy serves 1..%d" % (n, policy.max_batch))
        self.policy, self.queue, self.n, self.T = policy, queue, n, int(T)
        self._r = C.c_void_p()
        N.check(self._rfn("create")(policy._h, queue._q, n, C.byref(self._r)))
        live = [(p, r) for p, r in getattr(policy, "_recorder_handles", ()) if r.value]
        policy._recorder_handles = live + [(self._prefix(), self._r)]

    def _rfn(self, name):
        return getattr(N.lib, "drl_%s_recorder_%s" % (self._prefix(), name))

    def close(self):
        if getattr(self, "_r", None) is not None:
            _destroy_recorder(self._prefix(), self._r)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check_rows(self, n):
        if n != self.n:
            raise ValueError("recorder act: %d rows, the recorder records %d" % (n, self.n))

    def reset(self):
        """Discard the steps recorded since the last commit (an unroll abandoned half-way); the next act is step 0."""
        N.check(self._rfn("reset")(self._r))

    def commit(self, reward, done, timeout_ms=-1):
        """Moves the n recorded records into the queue; reward float32 [n, T], done bool / uint8 [n, T]."""
        rw = N.as_c(reward, np.float32, (self.n, self.T), "reward")
        dn = N.as_c(N.as_u8(done), np.uint8, (self.n, self.T), "done")
        N.check(self._rfn("commit")(self._r, N.ptr(rw), N.ptr(dn), int(timeout_ms)))
