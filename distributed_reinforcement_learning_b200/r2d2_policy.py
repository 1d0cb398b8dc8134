"""Thin object wrapper over the ``drl_r2d2_policy_*`` C-ABI (include/drl_b200.h): the R2D2 policy engine.

One ``NativeR2D2Policy`` serves the actor loop of ``train_r2d2.py:167-251`` for up to 64 environments per call: one
batched ``Agent.get_action`` (agent/r2d2.py:171-191) on its own CUDA stream next to a training ``NativeR2D2Learner``,
and ``parameter_sync`` device to device from that learner.  The epsilon-greedy draws come from numpy's global stream on
the host, exactly as the reference makes them; the argmax and the selection run on the GPU.  It owns no target scope,
optimizer state, gradients or backward buffers.

``NativeR2D2Policy.recorder(queue, n)`` binds the engine to an ``R2D2DeviceFIFOQueue``: the recorder's ``act`` is the
engine's act that also writes the step's frames, previous actions and actions (and at step 0 h and c) into device
staging, and its ``commit`` moves the n recorded sequences into the queue without copying them through the host.
"""
import numpy as np

from . import _native as N
from .policy_handle import MAX_BATCH, PolicyHandle, RecorderHandle, explore_actions  # noqa: F401  (MAX_BATCH: rows per call)


class NativeR2D2Policy(PolicyHandle):
    prefix = "r2d2_policy"

    def __init__(self, max_batch, num_action=4, lstm_size=64, input_shape=(84, 84, 1), device=0, use_cuda_graph=True):
        h, w, c = input_shape
        self.max_batch, self.A, self.L = int(max_batch), int(num_action), int(lstm_size)
        self.input_shape = (int(h), int(w), int(c))
        self.device = int(device)
        self._create(N.R2d2PolicyConfig(self.max_batch, h, w, c, self.A, self.L, self.device,
                                        int(bool(use_cuda_graph))))

    def _learner_type(self):
        from .r2d2_learner import NativeR2D2Learner
        return NativeR2D2Learner

    def recorder(self, queue, n):
        """An ``R2D2PolicyRecorder`` of n rows (n <= max_batch) into ``queue`` (an ``R2D2DeviceFIFOQueue`` on this
        device)."""
        return R2D2PolicyRecorder(self, queue, n)

    # ---- inference -------------------------------------------------------------------
    def _act_args(self, state, previous_action, h, c, epsilon, explore_action):
        n, st, pa = self._inputs(state, previous_action)
        hh = N.as_c(h, np.float32, (n, self.L), "h")
        cc = N.as_c(c, np.float32, (n, self.L), "c")
        ex = self._explore(n, epsilon, explore_action)
        outs = (np.empty(n, np.int32), np.empty((n, self.A), np.float32), np.empty(n, np.float32),
                np.empty((n, self.L), np.float32), np.empty((n, self.L), np.float32))
        return n, (st, pa, hh, cc), ex, outs

    @staticmethod
    def _act_call(fn, handle, n, ins, ex, outs):
        N.check(fn(handle, *([n] if n is not None else []), *[N.ptr(a) for a in ins],
                   N.ptr(ex) if ex is not None else None, *[N.ptr(a) for a in outs]))
        action, q, qa, ho, co = outs
        return dict(action=action, q=q, q_action=qa, h=ho, c=co)

    def act(self, state, previous_action, h, c, epsilon=None, explore_action=None):
        """Batched Agent.get_action for n <= max_batch rows: state uint8 [n, 84, 84, C], previous_action [n], h, c
        float32 [n, 64].  With ``epsilon`` (scalar or [n]) the explore decisions and random actions are drawn from
        numpy's global stream (``explore_actions``); ``explore_action`` ([n] ints, -1 = greedy) gives them directly;
        with neither every row is greedy.  Returns dict(action, q, q_action, h, c)."""
        n, ins, ex, outs = self._act_args(state, previous_action, h, c, epsilon, explore_action)
        return self._act_call(N.lib.drl_r2d2_policy_act, self._h, n, ins, ex, outs)


class R2D2PolicyRecorder(RecorderHandle):
    """Records n rows of a ``NativeR2D2Policy``'s acts as sequences of ``queue.seq_len`` steps, on the device.

    ``act`` has ``NativeR2D2Policy.act``'s signature and return value; call it for steps t = 0 .. S-1 with exactly n
    rows, then ``commit(reward, done)`` with the [n, S] rewards and done flags the environments gave.  The commit moves
    the n sequences into the queue in row order (blocking while it is full; ``timeout_ms`` >= 0 raises ``TimeoutError_``
    with nothing changed) and starts the next unroll.  Each sequence stores the frames and previous actions the acts
    were given, the actions they chose, and the h and c given to the act of step 0.  Closing the policy closes its
    recorders; keep the queue open while a recorder is in use."""

    def __init__(self, policy, queue, n):
        from .distributed_queue.buffer_queue import R2D2DeviceFIFOQueue
        self._bind(policy, queue, R2D2DeviceFIFOQueue, n, getattr(queue, "seq_len", 0))

    def act(self, state, previous_action, h, c, epsilon=None, explore_action=None):
        """``NativeR2D2Policy.act`` of the recorder's n rows, recorded as the next step of the unroll."""
        n, ins, ex, outs = self.policy._act_args(state, previous_action, h, c, epsilon, explore_action)
        self._check_rows(n)
        return self.policy._act_call(N.lib.drl_r2d2_policy_recorder_act, self._r, None, ins, ex, outs)
