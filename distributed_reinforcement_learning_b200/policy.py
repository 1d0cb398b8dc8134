"""Thin object wrapper over the ``drl_policy_*`` C-ABI (include/drl_b200.h): the IMPALA policy engine.

One ``NativePolicy`` serves the actor loop of ``train_impala.py:132-194`` for up to 64 environments per call: one
batched ``get_policy_and_action`` (agent/impala.py:118-130) with the action drawn on the GPU, on its own CUDA stream
next to a training ``NativeLearner``, and ``parameter_sync`` (agent/impala.py:111-112) device to device from that
learner.  It owns no optimizer state, gradients or backward buffers.
"""
import ctypes as C

import numpy as np

from . import _native as N

MAX_BATCH = 64


class NativePolicy:
    def __init__(self, max_batch, num_action=18, lstm_hidden_size=256, input_shape=(84, 84, 4), device=0,
                 use_cuda_graph=True):
        h, w, c = input_shape
        self.max_batch, self.A, self.L = int(max_batch), int(num_action), int(lstm_hidden_size)
        self.input_shape = (int(h), int(w), int(c))
        self.device = int(device)
        cfg = N.PolicyConfig(self.max_batch, h, w, c, self.A, self.L, self.device, int(bool(use_cuda_graph)))
        self._h = C.c_void_p()
        N.check(N.lib.drl_policy_create(C.byref(cfg), C.byref(self._h)))
        n = C.c_int64()
        N.check(N.lib.drl_policy_param_count(self._h, C.byref(n)))
        self.param_count = int(n.value)

    # ---- lifetime ----------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            N.lib.drl_policy_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- parameters ------------------------------------------------------------------
    def set_params(self, flat):
        """Flat float32 vector in the learner's TF order (NativeLearner.get_params)."""
        a = N.as_c(flat, np.float32, (self.param_count,), "params")
        N.check(N.lib.drl_policy_set_params(self._h, N.ptr(a), a.size))

    def get_params(self):
        a = np.empty(self.param_count, np.float32)
        N.check(N.lib.drl_policy_get_params(self._h, N.ptr(a), a.size))
        return a

    def sync_from(self, learner):
        """parameter_sync from a NativeLearner on the same device: device-to-device copy of its parameters after all
        work enqueued on it so far (a step in flight included); the learner's next update waits for the copy."""
        from .learner import NativeLearner
        if not isinstance(learner, NativeLearner):
            raise TypeError("sync_from takes a NativeLearner, got %s" % type(learner).__name__)
        N.check(N.lib.drl_policy_sync_from_learner(self._h, learner._h))

    # ---- inference -------------------------------------------------------------------
    def act(self, state, previous_action, h, c, uniform=None):
        """Batched get_policy_and_action for n <= max_batch rows: state uint8 [n, 84, 84, 4], previous_action [n],
        h, c float32 [n, 256].  ``uniform`` (float64 [n] in [0, 1)) are the draws of the GPU sampler; without it they
        come from ``np.random.random_sample(n)``, the global stream the reference's ``np.random.choice`` reads.
        Returns dict(action, policy, max_prob, h, c)."""
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
        if pa.size and (pa.min() < 0 or pa.max() >= self.A):
            raise ValueError("previous_action: values must lie in [0, %d)" % self.A)
        hh = N.as_c(h, np.float32, (n, self.L), "h")
        cc = N.as_c(c, np.float32, (n, self.L), "c")
        if uniform is None:
            uniform = np.random.random_sample(n)
        u = N.as_c(uniform, np.float64, (n,), "uniform")
        if not np.all((u >= 0.0) & (u < 1.0)):
            raise ValueError("uniform: draws must lie in [0, 1)")
        action = np.empty(n, np.int32)
        pol = np.empty((n, self.A), np.float32)
        ho = np.empty((n, self.L), np.float32)
        co = np.empty((n, self.L), np.float32)
        N.check(N.lib.drl_policy_act(self._h, n, N.ptr(st), N.ptr(pa), N.ptr(hh), N.ptr(cc), N.ptr(u), N.ptr(action),
                                     N.ptr(pol), N.ptr(ho), N.ptr(co)))
        return dict(action=action, policy=pol, max_prob=pol.max(-1), h=ho, c=co)

    def last_act_ms(self):
        """Device time of the last act (input copy + kernels), from CUDA events on the policy's stream."""
        ms = C.c_float()
        N.check(N.lib.drl_policy_last_act_ms(self._h, C.byref(ms)))
        return float(ms.value)
