"""CPU tests of the R2D2 learner's n-step double-Q targets and mixed max / mean priorities (DESIGN.md section 22): the
float64 oracle (tests/r2d2_nstep_oracle.py) at its defaults against the executed reference, its n-step targets and
priorities against an explicit loop written here, five injected defects that the parity bar must catch, and the
validation of the three drl_r2d2_config fields, which needs no GPU."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import parity
import r2d2_nstep_oracle as no
from oracle import r2d2_torch as rt

S, BI, A = 12, 3, 4
NT = S - BI - 1
GAMMA = rt.DEFAULT_CFG["discount_factor"]


def _batch():
    """Four sequences; the dones of sequence 1 fall at position 0 (window t = 6), k - 1 (t = 3, n = 4) and past the
    horizon (t = 3, 4 against the done at 9) of n = 4 horizons; sequence 2 ends with two dones; sequence 3 is random."""
    b = rt.make_sequences(4, S=S, A=A, seed=11)
    d = np.zeros((4, S), bool)
    d[1, [6, 9]] = True
    d[2, [S - 2, S - 1]] = True
    d[3] = np.random.default_rng(5).random(S) < 0.3
    b["done"] = d
    return b


def _explicit_target(main_q, target_q, reward, done, n):
    """h(G) window by window, G written out as sum_j (prod_{l<j} D) r + (prod_{l<k} D) h^-1(Q_target[t+k][a*])."""
    B = reward.shape[0]
    out = np.zeros((B, NT))
    for b in range(B):
        for i in range(NT):
            t = BI + i
            k = min(n, S - 1 - t)
            D = [0.0 if done[b, t + l] else GAMMA for l in range(k)]
            a = int(np.argmax(main_q[b, t + k]))
            boot = float(rt.vf_rescale_inv(torch.tensor(float(target_q[b, t + k, a]), dtype=torch.float64)))
            G = sum(math.prod(D[:j]) * float(np.float32(reward[b, t + j])) for j in range(k)) + math.prod(D) * boot
            out[b, i] = float(rt.vf_rescale(torch.tensor(G, dtype=torch.float64)))
    return out


def _explicit_priority(diff, eta):
    return np.array([eta * max(abs(x) for x in row) + (1 - eta) * sum(abs(x) for x in row) / len(row) for row in diff])


@pytest.fixture(scope="module")
def params():
    return rt.init_params(0, torch.float32), rt.init_params(1, torch.float32)


@pytest.fixture(scope="module")
def one_step(params):
    """main_q, target_q and the one-step outputs of the oracle on _batch()."""
    b = _batch()
    L = rt.Learner(*params, torch.float64, seq_len=S, burn_in=BI)
    with torch.no_grad():
        o = L.losses(*[b[k] for k in rt.TRAIN_FIELDS[:-1]], weight=b["weight"])
    return b, o


def test_defaults_equal_the_executed_reference(params):
    """With n_step=1 and priority_eta=None the oracle is the restatement the executed reference pins
    (tests/test_oracle_refexec.py): the same fetches, gradients and three training steps."""
    import test_oracle_refexec as tr
    from oracle import ref_exec
    if not ref_exec.available():
        pytest.skip("the reference checkout is not present")
    Sx, bix = 6, 2
    b = rt.make_sequences(2, S=Sx, seed=2468)
    args = [b[k] for k in rt.TRAIN_FIELDS]
    R = ref_exec.ReferenceR2D2(*params, seq_len=Sx, burn_in=bix)
    f = R.fetch(args, list(tr.R2D2_FETCH))
    rg = R.gradients(R.feed(*args))
    L = no.Learner(*params, torch.float64, seq_len=Sx, burn_in=bix)
    out, g = L.gradients(*args[:7], weight=args[7])
    for k in tr.R2D2_FETCH:
        assert tr._rel(out[k].detach().numpy(), f[k]) < 1e-12, k
    for n in g:
        assert tr._rel(g[n].numpy(), rg[n]) < 1e-11, n
    for _ in range(3):
        r = R.agent.train(*args)
        r2 = L.train(*args)
        assert float(r[0]) == pytest.approx(r2[0], rel=1e-6) and tr._rel(np.asarray(r[1]), r2[1]) < 1e-5


def test_defaults_equal_the_base_oracle(params, one_step):
    b, o = one_step
    args = [b[k] for k in rt.TRAIN_FIELDS]
    base = rt.Learner(*params, torch.float64, seq_len=S, burn_in=BI).train(*args)
    mine = no.Learner(*params, torch.float64, seq_len=S, burn_in=BI).train(*args)
    assert base[0] == mine[0] and np.array_equal(base[1], mine[1])


@pytest.mark.parametrize("n", [1, 2, 4, NT])
def test_nstep_target_equals_the_explicit_loop(params, one_step, n):
    b, o = one_step
    L = no.Learner(*params, torch.float64, n_step=n, seq_len=S, burn_in=BI)
    with torch.no_grad():
        got = L.losses(*[b[k] for k in rt.TRAIN_FIELDS[:-1]], weight=b["weight"])
    mq, tq = o["main_q"].numpy(), o["target_q"].numpy()
    exp = _explicit_target(mq, tq, b["reward"], b["done"], n)
    assert np.max(np.abs(got["target_value"].numpy() - exp)) <= 1e-13 * max(1.0, np.max(np.abs(exp)))
    diff = exp - got["state_action_value"].numpy()
    w = b["weight"].astype(np.float64)
    assert float(got["value_loss"]) == pytest.approx(float(np.mean(w * (diff ** 2).mean(1))), rel=1e-13)
    if n == 1:       # the reference's target
        assert np.array_equal(got["target_value"].numpy(), o["target_value"].numpy())


def test_the_fixture_covers_the_horizon_cases():
    b = _batch()
    d = b["done"]
    n = 4
    at0 = atk1 = past = trunc = False
    for bb in range(4):
        for i in range(NT):
            t = BI + i
            k = min(n, S - 1 - t)
            trunc |= k < n
            pos = [l for l in range(S - t) if d[bb, t + l]]
            at0 |= 0 in pos
            atk1 |= (k - 1) in pos and k > 1
            past |= any(p >= k for p in pos) and not any(p < k for p in pos)
    assert at0 and atk1 and past and trunc


@pytest.mark.parametrize("eta", [None, 0.0, 0.9, 1.0])
def test_priority_equals_the_explicit_rule(params, one_step, eta):
    b, o = one_step
    args = [b[k] for k in rt.TRAIN_FIELDS]
    L = no.Learner(*params, torch.float64, n_step=3, priority_eta=eta, seq_len=S, burn_in=BI)
    res, out, _, _ = L.train(*args, return_all=True)
    diff = out["target_value"].numpy() - out["state_action_value"].detach().numpy()
    exp = np.abs(diff.mean(1)) if eta is None else _explicit_priority(diff, eta)
    assert np.max(np.abs(res[1] - exp)) <= 1e-14 * max(1.0, np.max(exp))
    one = no.Learner(*params, torch.float64, n_step=3, priority_eta=eta, seq_len=S, burn_in=BI)
    row = [b[k][2] for k in rt.TRAIN_FIELDS[:-1]]
    assert one.get_td_error(*row) == pytest.approx(float(exp[2]), rel=1e-12)


# ---- injected defects -------------------------------------------------------------------------------------------------

def _defect_target(mq, tq, reward, done, n, bug):
    B = reward.shape[0]
    out = np.zeros((B, NT))
    h = lambda x: float(rt.vf_rescale(torch.tensor(x, dtype=torch.float64)))        # noqa: E731
    hinv = lambda x: float(rt.vf_rescale_inv(torch.tensor(x, dtype=torch.float64)))  # noqa: E731
    # horizon_not_truncated: every window takes n steps, read through the flat batch-major index b S + t + j, so a
    # horizon past S - 1 runs into the next sequence
    flat = lambda x, b, u: x[(b + u // S) % B, u % S]                                 # noqa: E731
    for b in range(B):
        for i in range(NT):
            t = BI + i
            k = n if bug == "horizon_not_truncated" else min(n, S - 1 - t)
            D = [0.0 if flat(done, b, t + l) else GAMMA for l in range(k)]
            a = int(np.argmax(flat(tq if bug == "argmax_on_target" else mq, b, t + k)))
            boot = float(flat(tq, b, t + k)[a])
            R = [float(np.float32(flat(reward, b, t + j))) for j in range(k)]
            if bug == "bootstrap_not_cut":
                G = sum(math.prod(D[:j]) * R[j] for j in range(k)) + GAMMA ** k * hinv(boot)
                out[b, i] = h(G)
            elif bug == "h_per_reward":
                out[b, i] = sum(math.prod(D[:j]) * h(R[j]) for j in range(k)) + math.prod(D) * boot
            else:
                G = sum(math.prod(D[:j]) * R[j] for j in range(k)) + math.prod(D) * hinv(boot)
                out[b, i] = h(G)
    return out


@pytest.mark.parametrize("bug", ["bootstrap_not_cut", "horizon_not_truncated", "argmax_on_target", "h_per_reward"])
def test_each_target_defect_misses_its_row_by_10x(one_step, bug):
    b, o = one_step
    mq, tq = o["main_q"].numpy(), o["target_q"].numpy()
    ok = _defect_target(mq, tq, b["reward"], b["done"], 4, None)
    assert np.max(np.abs(ok - _explicit_target(mq, tq, b["reward"], b["done"], 4))) < 1e-12
    err = parity.rel_err(_defect_target(mq, tq, b["reward"], b["done"], 4, bug), ok)
    assert err >= 10 * parity.TOL, (bug, err)


def test_signed_mean_priority_misses_its_row_by_10x(one_step):
    b, o = one_step
    diff = o["target_value"].numpy() - o["state_action_value"].numpy()
    eta = 0.9
    bad = eta * np.abs(diff).max(1) + (1 - eta) * np.abs(diff.mean(1))
    err = parity.rel_err(bad, no.priority(diff, eta))
    assert err >= 10 * parity.TOL, err


# ---- drl_r2d2_config validation -----------------------------------------------------------------------------------------

def _config(**kw):
    from distributed_reinforcement_learning_b200 import _native as N
    cfg = N.R2d2Config(4, 80, 40, 84, 84, 1, 4, 64, 0.997, 1e-4, 99, 2, 0, 0)
    for k, v in kw.items():
        setattr(cfg, k, v)
    return N, cfg


def _create(**kw):
    N, cfg = _config(**kw)
    h = C.c_void_p()
    return N, N.lib.drl_r2d2_create(C.byref(cfg), C.byref(h)), N.lib.drl_last_error().decode()


@pytest.mark.parametrize("n", [0, 1, 39])
def test_valid_n_step_reaches_the_device_lookup(n):
    """device 99 does not exist (with or without a GPU): a valid config fails at the device lookup, not before"""
    N, rc, msg = _create(n_step=n)
    assert rc == N.DRL_ERR_CUDA and "device 99" in msg


@pytest.mark.parametrize("n", [40, -1])
def test_n_step_outside_the_window_is_refused(n):
    N, rc, msg = _create(n_step=n)
    assert rc == N.DRL_ERR_INVALID and "n_step" in msg and "39" in msg


@pytest.mark.parametrize("eta", [-0.1, 1.1, float("nan"), float("inf")])
def test_priority_eta_outside_the_unit_interval_is_refused(eta):
    N, rc, msg = _create(priority_rule=1, priority_eta=eta)
    assert rc == N.DRL_ERR_INVALID and "priority_eta" in msg and "[0, 1]" in msg


@pytest.mark.parametrize("eta", [0.0, 0.9, 1.0])
def test_valid_priority_eta_reaches_the_device_lookup(eta):
    N, rc, msg = _create(priority_rule=1, priority_eta=eta)
    assert rc == N.DRL_ERR_CUDA


def test_eta_is_not_read_under_the_reference_rule():
    N, rc, msg = _create(priority_rule=0, priority_eta=float("nan"))
    assert rc == N.DRL_ERR_CUDA


@pytest.mark.parametrize("rule", [2, -1])
def test_unknown_priority_rule_is_refused(rule):
    N, rc, msg = _create(priority_rule=rule)
    assert rc == N.DRL_ERR_INVALID and "priority_rule" in msg


def test_agent_setters_check_their_ranges():
    from distributed_reinforcement_learning_b200.agent import r2d2
    a = r2d2.Agent(80, 40, [84, 84, 1], 4, 64, 0.997, 1e-4, 1e-4, 1e9, 40.0, "r2d2_nstep_ranges", "r2d2_nstep_ranges")
    for bad in (0, 40):
        with pytest.raises(ValueError, match="n_step"):
            a.set_n_step(bad)
    for bad in (-0.1, 1.1, float("nan")):
        with pytest.raises(ValueError, match="priority_eta"):
            a.set_priority_eta(bad)
    a.set_n_step(5)
    a.set_priority_eta(0.9)
    assert (a.n_step, a.priority_eta) == (5, 0.9)
