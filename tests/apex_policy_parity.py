"""Parity harness of the Ape-X / A3C policy engine: NativeApexPolicy.act against the float64 oracle's
``dueling_network`` (model/apex_value.py:22-41) and NativeA3CPolicy.act against ``a3c_torch.network``
(model/actor_critic.py:28-39), on the same float32 parameters and inputs.  Used by tests/test_gpu_apex_policy.py and
by ``__graft_entry__.smoke()``."""
import numpy as np
import torch

import parity
from oracle import a3c_torch as at
from oracle import apex_torch as ax

APEX, A3C = 0, 1


def make_params(seed, A, algo=APEX):
    """The oracle's init_params with small nonzero biases (the initial biases are zero)."""
    p = (ax if algo == APEX else at).init_params(seed, torch.float32, num_action=A)
    g = torch.Generator().manual_seed(seed + 1)
    for k in p:
        if k.endswith(".b"):
            p[k] = (torch.rand(p[k].shape, generator=g) - 0.5) * 0.2
    return p


flatten_params = ax.flatten_params


def make_inputs(n, A, seed):
    """n rows (state uint8 [n,84,84,4], previous_action) from the synthetic Ape-X transition generator."""
    t = ax.make_transitions(n, A=A, seed=seed)
    return np.ascontiguousarray(t["state"]), np.ascontiguousarray(t["previous_action"])


def _image(state):
    return torch.from_numpy((state.astype(np.float64) / 255).astype(np.float32)).double()


def oracle_act(params, state, previous_action, A, algo=APEX):
    """float64 forward on float32 parameters -> q (Ape-X) or policy (A3C) [n, A] as numpy."""
    p64 = {k: v.double() for k, v in params.items()}
    pa = torch.from_numpy(previous_action.astype(np.int64))
    with torch.no_grad():
        if algo == APEX:
            return ax.dueling_network(p64, _image(state), pa, A).numpy()
        return at.network(p64, _image(state), pa, A)[0].numpy()


def compare_act(pol, params, n, A, seed=7, **act_kw):
    """Runs pol.act on n synthetic rows and returns ({name: rel err vs the oracle}, act outputs)."""
    st, pa = make_inputs(n, A, seed)
    out = pol.act(st, pa, **act_kw)
    if pol.algo == APEX:
        return {"q": parity.rel_err(out["q"], oracle_act(params, st, pa, A, APEX))}, out
    return {"policy": parity.rel_err(out["policy"], oracle_act(params, st, pa, A, A3C))}, out


def expected_action(policy_row, u):
    """numpy.random.RandomState.choice(A, p=policy_row) for the uniform draw u (legacy generator)."""
    cdf = np.cumsum(np.asarray(policy_row, np.float64))
    cdf /= cdf[-1]
    return min(int(np.searchsorted(cdf, u, side="right")), len(cdf) - 1)
