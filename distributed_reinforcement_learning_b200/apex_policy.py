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
import numpy as np

from . import _native as N
from .policy_handle import MAX_BATCH, PolicyHandle, RecorderHandle  # noqa: F401  (MAX_BATCH: rows per call)

APEX, A3C = 0, 1


class _ApexPolicyBase(PolicyHandle):
    prefix = "apex_policy"
    algo = None

    def __init__(self, max_batch, num_action=4, input_shape=(84, 84, 4), device=0, use_cuda_graph=True):
        h, w, c = input_shape
        self.max_batch, self.A = int(max_batch), int(num_action)
        self.input_shape = (int(h), int(w), int(c))
        self.device = int(device)
        self._create(N.ApexPolicyConfig(self.max_batch, h, w, c, self.A, self.algo, self.device,
                                        int(bool(use_cuda_graph))))


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
        ex = self._explore(n, epsilon, explore_action)
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

    def recorder(self, queue, n):
        """An ``A3CPolicyRecorder`` of n rows (n <= max_batch) into ``queue`` (an ``A3CDeviceFIFOQueue`` on this
        device)."""
        return A3CPolicyRecorder(self, queue, n)

    def _act_args(self, state, previous_action, uniform):
        n, st, pa = self._inputs(state, previous_action)
        if uniform is None:
            uniform = np.random.random_sample(n)
        u = np.asarray(uniform)
        if not np.issubdtype(u.dtype, np.floating):
            raise ValueError("uniform: expected floats, got %s" % u.dtype)
        u = N.as_c(u, np.float64, (n,), "uniform")
        if not ((u >= 0.0) & (u < 1.0)).all():
            raise ValueError("uniform: values must lie in [0, 1)")
        outs = (np.empty(n, np.int32), np.empty((n, self.A), np.float32), np.empty(n, np.float32))
        return n, st, pa, u, outs

    def act(self, state, previous_action, uniform=None):
        """Batched get_policy_and_action for n <= max_batch rows: state uint8 [n, 84, 84, 4], previous_action [n].
        Row i's action is what ``np.random.choice(A, p=policy[i])`` picks for the uniform draw ``uniform[i]`` in
        [0, 1); by default the draws are ``np.random.random_sample(n)``, the stream that choice reads.
        Returns dict(action, policy, max_prob) with max_prob = policy[action] (the reference's name for it)."""
        n, st, pa, u, (action, policy, prob) = self._act_args(state, previous_action, uniform)
        N.check(N.lib.drl_a3c_policy_act(self._h, n, N.ptr(st), N.ptr(pa), N.ptr(u), N.ptr(action), N.ptr(policy),
                                         N.ptr(prob)))
        return dict(action=action, policy=policy, max_prob=prob)


class A3CPolicyRecorder(RecorderHandle):
    """Records n rows of a ``NativeA3CPolicy``'s acts as unrolls of ``queue.trajectory`` steps, on the device.

    ``act`` is ``NativeA3CPolicy.act`` plus ``previous_next_state``: the [n] frames ``env.step`` returned at the
    previous step (ignored at step 0).  Call it for steps t = 0 .. T-1 with exactly n rows, then ``commit(reward, done,
    next_state)`` with the [n, T] rewards and done flags and the [n] frames of step T-1.  The commit moves the n unrolls
    into the queue in row order (blocking while it is full; ``timeout_ms`` >= 0 raises ``TimeoutError_`` with nothing
    changed) and starts the next unroll.  Each unroll stores the frames and previous actions the acts were given, the
    actions they chose, and as next_state row t the frame of step t + 1 (or, after an episode reset, the
    ``previous_next_state`` given; or, at T-1, the commit's).  Closing the policy closes its recorders; keep the queue
    open while a recorder is in use."""
    prefix = "a3c_policy"

    def __init__(self, policy, queue, n):
        from .distributed_queue.buffer_queue import A3CDeviceFIFOQueue
        self._bind(policy, queue, A3CDeviceFIFOQueue, n, getattr(queue, "trajectory", 0))

    def _frames(self, frames, name):
        return N.as_c(frames, np.uint8, (self.n,) + self.policy.input_shape, name)

    def act(self, state, previous_action, uniform=None, previous_next_state=None):
        """``NativeA3CPolicy.act`` of the recorder's n rows, recorded as the next step of the unroll."""
        n, st, pa, u, (action, policy, prob) = self.policy._act_args(state, previous_action, uniform)
        self._check_rows(n)
        pn = None if previous_next_state is None else self._frames(previous_next_state, "previous_next_state")
        N.check(self._rfn("act")(self._r, N.ptr(st), N.ptr(pa), N.ptr(u),
                                                  N.ptr(pn) if pn is not None else None, N.ptr(action),
                                                  N.ptr(policy), N.ptr(prob)))
        return dict(action=action, policy=policy, max_prob=prob)

    def commit(self, reward, done, next_state, timeout_ms=-1):
        """Moves the n recorded unrolls into the queue; reward float32 [n, T], done bool / uint8 [n, T], next_state
        uint8 [n, 84, 84, 4] (the frames of step T-1)."""
        rw = N.as_c(reward, np.float32, (self.n, self.T), "reward")
        dn = N.as_c(N.as_u8(done), np.uint8, (self.n, self.T), "done")
        ns = self._frames(next_state, "next_state")
        N.check(self._rfn("commit")(self._r, N.ptr(rw), N.ptr(dn), N.ptr(ns), int(timeout_ms)))
