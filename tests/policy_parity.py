"""Parity harness of the policy engine: NativePolicy.act against the float64 oracle's ``network``
(model/impala_actor_critic.py:33-42) on the same float32 parameters and inputs.  Used by tests/test_gpu_policy.py and by
``__graft_entry__.smoke()``."""
import numpy as np
import torch

import parity
from oracle import impala_torch as it


def make_inputs(n, A, seed):
    """n single-step rows (state, previous_action, h, c) from the synthetic learner batch generator."""
    batch, _, _ = parity.make_case(n, 3, A, seed=seed)
    return (np.ascontiguousarray(batch["state"][:, 0]), np.ascontiguousarray(batch["previous_action"][:, 0]),
            np.ascontiguousarray(batch["initial_h"][:, 0]), np.ascontiguousarray(batch["initial_c"][:, 0]))


def oracle_act(params, state, previous_action, h, c, A):
    """float64 network() on float32 parameters -> (policy, h', c') as numpy."""
    p64 = {k: v.double() for k, v in params.items()}
    x = torch.from_numpy((state.astype(np.float64) / 255).astype(np.float32)).double()
    a, _, cc, hh = it.network(p64, x, torch.from_numpy(previous_action.astype(np.int64)), torch.from_numpy(h).double(),
                              torch.from_numpy(c).double(), A, 256)
    return a.numpy(), hh.numpy(), cc.numpy()


def compare_act(pol, params, n, A, seed=7, uniform=None):
    """Runs pol.act on n synthetic rows and returns ({name: rel err vs the oracle}, act outputs)."""
    st, pa, h, c = make_inputs(n, A, seed)
    out = pol.act(st, pa, h, c, uniform=uniform)
    ra, rh, rc = oracle_act(params, st, pa, h, c, A)
    errs = {"policy": parity.rel_err(out["policy"], ra), "h": parity.rel_err(out["h"], rh),
            "c": parity.rel_err(out["c"], rc)}
    return errs, out


def expected_action(policy_row, u):
    """numpy.random.RandomState.choice(A, p=policy_row) for the uniform draw u (legacy generator)."""
    cdf = np.cumsum(np.asarray(policy_row, np.float64))
    cdf /= cdf[-1]
    return min(int(np.searchsorted(cdf, u, side="right")), len(cdf) - 1)
