"""Parity harness of the R2D2 policy engine: NativeR2D2Policy.act against the float64 oracle's ``network``
(model/r2d2_lstm.py:28-53, through ``r2d2_torch.Learner.step_q``) on the same float32 parameters and inputs.  Used by
tests/test_gpu_r2d2_policy.py and by ``__graft_entry__.smoke()``."""
import numpy as np
import torch

import parity
from oracle import r2d2_torch as rt


def make_params(seed, A, C=1):
    """r2d2_torch.init_params with small nonzero biases (the initial biases are zero)."""
    p = rt.init_params(seed, torch.float32, num_action=A, input_shape=(84, 84, C))
    g = torch.Generator().manual_seed(seed + 1)
    for k in p:
        if k.endswith(".b"):
            p[k] = (torch.rand(p[k].shape, generator=g) - 0.5) * 0.2
    return p


def make_inputs(n, A, C, seed):
    """n single-step rows (state, previous_action, h, c) from the synthetic R2D2 sequence generator."""
    b = rt.make_sequences(n, S=1, A=A, input_shape=(84, 84, C), seed=seed)
    return (np.ascontiguousarray(b["state"][:, 0]), np.ascontiguousarray(b["previous_action"][:, 0]),
            np.ascontiguousarray(b["h"][:, 0]), np.ascontiguousarray(b["c"][:, 0]))


def oracle_act(params, state, previous_action, h, c, A, C=1):
    """float64 Agent.get_action network step on float32 parameters -> (q, h', c') as numpy."""
    L = rt.Learner(params, params, torch.float64, num_action=A, input_shape=(84, 84, C))
    return L.step_q(state, h, c, previous_action)


def compare_act(pol, params, n, A, C=1, seed=7, **act_kw):
    """Runs pol.act on n synthetic rows and returns ({name: rel err vs the oracle}, act outputs)."""
    st, pa, h, c = make_inputs(n, A, C, seed)
    out = pol.act(st, pa, h, c, **act_kw)
    q, hh, cc = oracle_act(params, st, pa, h, c, A, C)
    errs = {"q": parity.rel_err(out["q"], q), "h": parity.rel_err(out["h"], hh), "c": parity.rel_err(out["c"], cc)}
    return errs, out
