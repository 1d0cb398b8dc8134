"""Thin object wrapper over the ``drl_r2d2_policy_*`` C-ABI (include/drl_b200.h): the R2D2 policy engine.

One ``NativeR2D2Policy`` serves the actor loop of ``train_r2d2.py:167-251`` for up to 64 environments per call: one
batched ``Agent.get_action`` (agent/r2d2.py:171-191) on its own CUDA stream next to a training ``NativeR2D2Learner``,
and ``parameter_sync`` device to device from that learner.  The epsilon-greedy draws come from numpy's global stream on
the host, exactly as the reference makes them; the argmax and the selection run on the GPU.  It owns no target scope,
optimizer state, gradients or backward buffers.
"""
import numpy as np

from . import _native as N
from .policy_handle import MAX_BATCH, PolicyHandle, explore_actions  # noqa: F401  (MAX_BATCH: rows per call)


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

    # ---- inference -------------------------------------------------------------------
    def act(self, state, previous_action, h, c, epsilon=None, explore_action=None):
        """Batched Agent.get_action for n <= max_batch rows: state uint8 [n, 84, 84, C], previous_action [n], h, c
        float32 [n, 64].  With ``epsilon`` (scalar or [n]) the explore decisions and random actions are drawn from
        numpy's global stream (``explore_actions``); ``explore_action`` ([n] ints, -1 = greedy) gives them directly;
        with neither every row is greedy.  Returns dict(action, q, q_action, h, c)."""
        n, st, pa = self._inputs(state, previous_action)
        hh = N.as_c(h, np.float32, (n, self.L), "h")
        cc = N.as_c(c, np.float32, (n, self.L), "c")
        ex = self._explore(n, epsilon, explore_action)
        action = np.empty(n, np.int32)
        q = np.empty((n, self.A), np.float32)
        qa = np.empty(n, np.float32)
        ho = np.empty((n, self.L), np.float32)
        co = np.empty((n, self.L), np.float32)
        N.check(N.lib.drl_r2d2_policy_act(self._h, n, N.ptr(st), N.ptr(pa), N.ptr(hh), N.ptr(cc),
                                          N.ptr(ex) if ex is not None else None, N.ptr(action), N.ptr(q), N.ptr(qa),
                                          N.ptr(ho), N.ptr(co)))
        return dict(action=action, q=q, q_action=qa, h=ho, c=co)
