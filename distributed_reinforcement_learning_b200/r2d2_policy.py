"""Thin object wrapper over the ``drl_r2d2_policy_*`` C-ABI (include/drl_b200.h): the R2D2 policy engine.

One ``NativeR2D2Policy`` serves the actor loop of ``train_r2d2.py:167-251`` for up to 64 environments per call: one
batched ``Agent.get_action`` (agent/r2d2.py:171-191) on its own CUDA stream next to a training ``NativeR2D2Learner``,
and ``parameter_sync`` device to device from that learner.  The epsilon-greedy draws come from numpy's global stream on
the host, exactly as the reference makes them; the argmax and the selection run on the GPU.  It owns no target scope,
optimizer state, gradients or backward buffers.
"""
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


class NativeR2D2Policy:
    def __init__(self, max_batch, num_action=4, lstm_size=64, input_shape=(84, 84, 1), device=0, use_cuda_graph=True):
        h, w, c = input_shape
        self.max_batch, self.A, self.L = int(max_batch), int(num_action), int(lstm_size)
        self.input_shape = (int(h), int(w), int(c))
        self.device = int(device)
        cfg = N.R2d2PolicyConfig(self.max_batch, h, w, c, self.A, self.L, self.device, int(bool(use_cuda_graph)))
        self._h = C.c_void_p()
        N.check(N.lib.drl_r2d2_policy_create(C.byref(cfg), C.byref(self._h)))
        n = C.c_int64()
        N.check(N.lib.drl_r2d2_policy_param_count(self._h, C.byref(n)))
        self.param_count = int(n.value)

    # ---- lifetime ----------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            N.lib.drl_r2d2_policy_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- parameters ------------------------------------------------------------------
    def set_params(self, flat):
        """Flat float32 vector of the main scope in the learner's TF order (NativeR2D2Learner.get_params(MAIN))."""
        a = N.as_c(flat, np.float32, (self.param_count,), "params")
        N.check(N.lib.drl_r2d2_policy_set_params(self._h, N.ptr(a), a.size))

    def get_params(self):
        a = np.empty(self.param_count, np.float32)
        N.check(N.lib.drl_r2d2_policy_get_params(self._h, N.ptr(a), a.size))
        return a

    def sync_from(self, learner):
        """parameter_sync from a NativeR2D2Learner on the same device: device-to-device copy of its main parameters
        after all work enqueued on it so far (a step in flight included); the learner's next update waits for the copy."""
        from .r2d2_learner import NativeR2D2Learner
        if not isinstance(learner, NativeR2D2Learner):
            raise TypeError("sync_from takes a NativeR2D2Learner, got %s" % type(learner).__name__)
        N.check(N.lib.drl_r2d2_policy_sync_from_learner(self._h, learner._h))

    # ---- inference -------------------------------------------------------------------
    def act(self, state, previous_action, h, c, epsilon=None, explore_action=None):
        """Batched Agent.get_action for n <= max_batch rows: state uint8 [n, 84, 84, C], previous_action [n], h, c
        float32 [n, 64].  With ``epsilon`` (scalar or [n]) the explore decisions and random actions are drawn from
        numpy's global stream (``explore_actions``); ``explore_action`` ([n] ints, -1 = greedy) gives them directly;
        with neither every row is greedy.  Returns dict(action, q, q_action, h, c)."""
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
        hh = N.as_c(h, np.float32, (n, self.L), "h")
        cc = N.as_c(c, np.float32, (n, self.L), "c")
        if epsilon is not None and explore_action is not None:
            raise ValueError("pass epsilon or explore_action, not both")
        if epsilon is not None:
            explore_action = explore_actions(epsilon, n, self.A)
        ex = None
        if explore_action is not None:
            ex_in = np.asarray(explore_action)
            if not np.issubdtype(ex_in.dtype, np.integer):
                raise ValueError("explore_action: expected integers, got %s" % ex_in.dtype)
            ex = N.as_c(ex_in, np.int32, (n,), "explore_action")
            if ex.min() < -1 or ex.max() >= self.A:
                raise ValueError("explore_action: values must lie in [-1, %d)" % self.A)
        action = np.empty(n, np.int32)
        q = np.empty((n, self.A), np.float32)
        qa = np.empty(n, np.float32)
        ho = np.empty((n, self.L), np.float32)
        co = np.empty((n, self.L), np.float32)
        N.check(N.lib.drl_r2d2_policy_act(self._h, n, N.ptr(st), N.ptr(pa), N.ptr(hh), N.ptr(cc),
                                          N.ptr(ex) if ex is not None else None, N.ptr(action), N.ptr(q), N.ptr(qa),
                                          N.ptr(ho), N.ptr(co)))
        return dict(action=action, q=q, q_action=qa, h=ho, c=co)

    def last_act_ms(self):
        """Device time of the last act (input copy + kernels), from CUDA events on the policy's stream."""
        ms = C.c_float()
        N.check(N.lib.drl_r2d2_policy_last_act_ms(self._h, C.byref(ms)))
        return float(ms.value)
