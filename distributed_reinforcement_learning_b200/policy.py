"""Thin object wrapper over the ``drl_policy_*`` C-ABI (include/drl_b200.h): the IMPALA policy engine.

One ``NativePolicy`` serves the actor loop of ``train_impala.py:132-194`` for up to 64 environments per call: one
batched ``get_policy_and_action`` (agent/impala.py:118-130) with the action drawn on the GPU, on its own CUDA stream
next to a training ``NativeLearner``, and ``parameter_sync`` (agent/impala.py:111-112) device to device from that
learner.  It owns no optimizer state, gradients or backward buffers.

``NativePolicy.recorder(queue, n)`` binds the engine to a ``DeviceFIFOQueue``: the recorder's ``act`` is the engine's
act that also writes the step's frames, previous actions, h, c, policies and actions into device staging, and its
``commit`` moves the n recorded trajectories into the queue without copying them through the host.
"""
import numpy as np

from . import _native as N
from .policy_handle import MAX_BATCH, PolicyHandle, RecorderHandle  # noqa: F401  (MAX_BATCH: rows per call)


class NativePolicy(PolicyHandle):
    prefix = "policy"

    def __init__(self, max_batch, num_action=18, lstm_hidden_size=256, input_shape=(84, 84, 4), device=0,
                 use_cuda_graph=True):
        h, w, c = input_shape
        self.max_batch, self.A, self.L = int(max_batch), int(num_action), int(lstm_hidden_size)
        self.input_shape = (int(h), int(w), int(c))
        self.device = int(device)
        self._create(N.PolicyConfig(self.max_batch, h, w, c, self.A, self.L, self.device, int(bool(use_cuda_graph))))

    def _learner_type(self):
        from .learner import NativeLearner
        return NativeLearner

    def recorder(self, queue, n):
        """A ``PolicyRecorder`` of n rows (n <= max_batch) into ``queue`` (a ``DeviceFIFOQueue`` on this device)."""
        return PolicyRecorder(self, queue, n)

    # ---- inference -------------------------------------------------------------------
    def _act_args(self, state, previous_action, h, c, uniform):
        n, st, pa = self._inputs(state, previous_action)
        hh = N.as_c(h, np.float32, (n, self.L), "h")
        cc = N.as_c(c, np.float32, (n, self.L), "c")
        if uniform is None:
            uniform = np.random.random_sample(n)
        u = N.as_c(uniform, np.float64, (n,), "uniform")
        if not np.all((u >= 0.0) & (u < 1.0)):
            raise ValueError("uniform: draws must lie in [0, 1)")
        outs = (np.empty(n, np.int32), np.empty((n, self.A), np.float32), np.empty((n, self.L), np.float32),
                np.empty((n, self.L), np.float32))
        return n, (st, pa, hh, cc, u), outs

    @staticmethod
    def _act_result(outs):
        action, pol, ho, co = outs
        return dict(action=action, policy=pol, max_prob=pol.max(-1), h=ho, c=co)

    def act(self, state, previous_action, h, c, uniform=None):
        """Batched get_policy_and_action for n <= max_batch rows: state uint8 [n, 84, 84, 4], previous_action [n],
        h, c float32 [n, 256].  ``uniform`` (float64 [n] in [0, 1)) are the draws of the GPU sampler; without it they
        come from ``np.random.random_sample(n)``, the global stream the reference's ``np.random.choice`` reads.
        Returns dict(action, policy, max_prob, h, c)."""
        n, ins, outs = self._act_args(state, previous_action, h, c, uniform)
        N.check(N.lib.drl_policy_act(self._h, n, *[N.ptr(a) for a in ins + outs]))
        return self._act_result(outs)


class PolicyRecorder(RecorderHandle):
    """Records n rows of a ``NativePolicy``'s acts as trajectories of ``queue.trajectory`` steps, on the device.

    ``act`` has ``NativePolicy.act``'s signature and return value; call it for steps t = 0 .. T-1 with exactly n rows,
    then ``commit(reward, done)`` with the [n, T] rewards and done flags the environments gave.  The commit moves the n
    trajectories into the queue in row order (blocking while it is full; ``timeout_ms`` >= 0 raises
    ``TimeoutError_`` with nothing changed) and starts the next unroll.  Each trajectory stores the frames, previous
    actions, h and c the acts were given and the policies and actions they returned.  Closing the policy closes its
    recorders; keep the queue open while a recorder is in use."""

    def __init__(self, policy, queue, n):
        from .distributed_queue.buffer_queue import DeviceFIFOQueue
        self._bind(policy, queue, DeviceFIFOQueue, n, getattr(queue, "trajectory", 0))

    def act(self, state, previous_action, h, c, uniform=None):
        """``NativePolicy.act`` of the recorder's n rows, recorded as the next step of the unroll."""
        n, ins, outs = self.policy._act_args(state, previous_action, h, c, uniform)
        self._check_rows(n)
        N.check(N.lib.drl_policy_recorder_act(self._r, *[N.ptr(a) for a in ins + outs]))
        return self.policy._act_result(outs)
