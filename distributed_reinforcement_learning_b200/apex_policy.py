"""Thin object wrappers over the ``drl_apex_policy_*`` C-ABI (include/drl_b200.h): the Ape-X and A3C policy engine.

The two families share the network body and the learner handle, so one engine serves both; only the action rule
differs.  ``NativeApexPolicy`` serves the actor loop of ``train_apex.py:157-231`` (one batched
``apex.Agent.get_policy_and_action``, agent/apex.py:88-102) and ``NativeA3CPolicy`` that of ``train_a3c.py:112-183``
(``a3c.Agent.get_policy_and_action``, agent/a3c.py:109-119), for up to 64 environments per call, on their own CUDA
stream next to a training ``NativeApexLearner`` / ``NativeA3CLearner``, with ``parameter_sync`` device to device from
that learner.  The random draws come from numpy's global stream on the host, exactly as the reference makes them; the
forward pass and the action selection run on the GPU.  Neither owns a target network, optimizer state, gradients or
backward buffers.
"""
import ctypes as C

import numpy as np

from . import _native as N
from .r2d2_policy import explore_actions

MAX_BATCH = 64
APEX, A3C = 0, 1


class _ApexPolicyBase:
    algo = None

    def __init__(self, max_batch, num_action=4, input_shape=(84, 84, 4), device=0, use_cuda_graph=True):
        h, w, c = input_shape
        self.max_batch, self.A = int(max_batch), int(num_action)
        self.input_shape = (int(h), int(w), int(c))
        self.device = int(device)
        cfg = N.ApexPolicyConfig(self.max_batch, h, w, c, self.A, self.algo, self.device, int(bool(use_cuda_graph)))
        self._h = C.c_void_p()
        N.check(N.lib.drl_apex_policy_create(C.byref(cfg), C.byref(self._h)))
        n = C.c_int64()
        N.check(N.lib.drl_apex_policy_param_count(self._h, C.byref(n)))
        self.param_count = int(n.value)

    # ---- lifetime ----------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            N.lib.drl_apex_policy_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- parameters ------------------------------------------------------------------
    def set_params(self, flat):
        """Flat float32 vector of one network in the learner's TF order (NativeApexLearner.get_params(MAIN),
        NativeA3CLearner.get_params())."""
        a = N.as_c(flat, np.float32, (self.param_count,), "params")
        N.check(N.lib.drl_apex_policy_set_params(self._h, N.ptr(a), a.size))

    def get_params(self):
        a = np.empty(self.param_count, np.float32)
        N.check(N.lib.drl_apex_policy_get_params(self._h, N.ptr(a), a.size))
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
        N.check(N.lib.drl_apex_policy_sync_from_learner(self._h, learner._h))

    def last_act_ms(self):
        """Device time of the last act (input copy + kernels), from CUDA events on the policy's stream."""
        ms = C.c_float()
        N.check(N.lib.drl_apex_policy_last_act_ms(self._h, C.byref(ms)))
        return float(ms.value)

    # ---- inputs ----------------------------------------------------------------------
    def _inputs(self, state, previous_action):
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


class NativeApexPolicy(_ApexPolicyBase):
    """The Ape-X engine (algo 0)."""
    algo = APEX

    def _learner_type(self):
        from .apex_learner import NativeApexLearner
        return NativeApexLearner

    def act(self, state, previous_action, epsilon=None, explore_action=None):
        """Batched get_policy_and_action for n <= max_batch rows: state uint8 [n, 84, 84, 4], previous_action [n].
        With ``epsilon`` (scalar or [n]) the explore decisions and random actions are drawn from numpy's global stream
        row by row (``r2d2_policy.explore_actions``: ``np.random.rand() > eps``, then ``np.random.choice(A)``);
        ``explore_action`` ([n] ints, -1 = greedy) gives them directly; with neither every row is greedy.
        Returns dict(action, q, q_action) with q_action = q[action]."""
        n, st, pa = self._inputs(state, previous_action)
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
        N.check(N.lib.drl_apex_policy_act(self._h, n, N.ptr(st), N.ptr(pa), N.ptr(ex) if ex is not None else None,
                                          N.ptr(action), N.ptr(q), N.ptr(qa)))
        return dict(action=action, q=q, q_action=qa)


class NativeA3CPolicy(_ApexPolicyBase):
    """The A3C engine (algo 1)."""
    algo = A3C

    def _learner_type(self):
        from .a3c_learner import NativeA3CLearner
        return NativeA3CLearner

    def act(self, state, previous_action, uniform=None):
        """Batched get_policy_and_action for n <= max_batch rows: state uint8 [n, 84, 84, 4], previous_action [n].
        Row i's action is what ``np.random.choice(A, p=policy[i])`` picks for the uniform draw ``uniform[i]`` in
        [0, 1); by default the draws are ``np.random.random_sample(n)``, the stream that choice reads.
        Returns dict(action, policy, max_prob) with max_prob = policy[action] (the reference's name for it)."""
        n, st, pa = self._inputs(state, previous_action)
        if uniform is None:
            uniform = np.random.random_sample(n)
        u = np.asarray(uniform)
        if not np.issubdtype(u.dtype, np.floating):
            raise ValueError("uniform: expected floats, got %s" % u.dtype)
        u = N.as_c(u, np.float64, (n,), "uniform")
        if not ((u >= 0.0) & (u < 1.0)).all():
            raise ValueError("uniform: values must lie in [0, 1)")
        action = np.empty(n, np.int32)
        policy = np.empty((n, self.A), np.float32)
        prob = np.empty(n, np.float32)
        N.check(N.lib.drl_a3c_policy_act(self._h, n, N.ptr(st), N.ptr(pa), N.ptr(u), N.ptr(action), N.ptr(policy),
                                         N.ptr(prob)))
        return dict(action=action, policy=policy, max_prob=prob)
