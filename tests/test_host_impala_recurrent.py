"""CPU (no GPU needed): the float64 oracle of the IMPALA learner's recurrent mode (tests/impala_recurrent_oracle.py) --
its gradients against finite differences, its identity with the stored-state oracle on trajectories an actor recorded
under the same parameters, each injected defect failing its row by 10x the parity bar -- and the create-time checks of
the new ``recurrent`` config field, which run before any device lookup."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import impala_torch as it
from oracle import synthetic

import impala_recurrent_oracle as ro

B, T, A, L = 3, 6, 5, 256


def _actor_batch(params, seed=3, life_loss=((0, 0), (1, 2), (2, T - 1)), episode_end=((0, 3), (2, 1))):
    """A batch recorded the way the reference actor records it (train_impala.py:149-181), by the single-step float64
    oracle network: (h, c) recorded before each step, kept across a life-loss done and zeroed after an episode end.
    Returns the batch and the records in float64 (the carried values exactly)."""
    batch = synthetic.make_batch(B, T=T, A=A, seed=seed)
    done = np.zeros((B, T), bool)
    end = np.zeros((B, T), bool)
    for b, t in life_loss:
        done[b, t] = True
    for b, t in episode_end:
        done[b, t] = end[b, t] = True
    p = {k: v.to(torch.float64) for k, v in params.items()}
    x = torch.from_numpy((batch["state"].astype(np.float64) / 255).astype(np.float32)).to(torch.float64)
    pa = torch.from_numpy(batch["previous_action"].astype(np.int64))
    h = torch.from_numpy(batch["initial_h"][:, 0]).to(torch.float64)
    c = torch.from_numpy(batch["initial_c"][:, 0]).to(torch.float64)
    hs, cs = torch.zeros(B, T, L, dtype=torch.float64), torch.zeros(B, T, L, dtype=torch.float64)
    with torch.no_grad():
        for t in range(T):
            hs[:, t], cs[:, t] = h, c
            _, _, c, h = it.network(p, x[:, t], pa[:, t], h, c, A, L)
            zero = torch.from_numpy(end[:, t])[:, None]
            h, c = torch.where(zero, torch.zeros_like(h), h), torch.where(zero, torch.zeros_like(c), c)
    batch = dict(batch, done=done, initial_h=hs.numpy().astype(np.float32), initial_c=cs.numpy().astype(np.float32))
    return batch, hs, cs


@pytest.fixture(scope="module")
def params():
    return it.init_params(0, torch.float32, num_action=A)


def _forward(learner, batch, hs, cs):
    """losses and taps of ``learner`` with the float64 records fed as they are (not rounded to float32)"""
    t = learner._prep(*[batch[k] for k in synthetic.TRAIN_FIELDS])
    t["h0"], t["c0"] = hs, cs
    windows, taps = learner._unrolled(t)
    return dict(it.loss_terms(learner.cfg, t, *windows), taps=taps)


def test_recurrent_forward_equals_stored_state_on_actor_recorded_trajectories(params):
    """Same parameters as the actor, dones at t = 0, in the middle and at t = T - 1, life losses (state kept) and
    episode ends (state zeroed): the unroll restarts exactly where the actor's state changed, so it equals the
    stored-state forward to float64 rounding."""
    batch, hs, cs = _actor_batch(params)
    rec = _forward(ro.RecurrentLearner(params, trajectory=T, num_action=A), batch, hs, cs)
    ref = _forward(it.Learner(params, torch.float64, "dedup", trajectory=T, num_action=A), batch, hs, cs)
    for k in ("pi_loss", "baseline_loss", "entropy", "total_loss"):
        r, f = float(rec[k].detach()), float(ref[k].detach())
        assert abs(r - f) <= 1e-12 * max(abs(f), 1.0), k
    for k in ("policy", "value", "h1", "c1"):
        np.testing.assert_allclose(rec["taps"][k].detach().numpy(), ref["taps"][k].detach().numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(rec["taps"]["hin"].detach().numpy(), hs.numpy(), rtol=0, atol=1e-12)


def test_recurrent_gradients_match_finite_differences(params):
    """d/dθ of a smooth function of the unrolled policy and value (no stop-gradient, unlike the V-trace losses) by
    central differences, at entries of the W_x and W_h rows of the LSTM kernel, its bias and the first head layers."""
    batch = ro.with_dones(synthetic.make_batch(2, T=5, A=A, seed=9), [(0, 1), (1, 0), (1, 3)])
    lr = ro.RecurrentLearner(params, trajectory=5, num_action=A)
    t = lr._prep(*[batch[k] for k in synthetic.TRAIN_FIELDS])
    g = torch.Generator().manual_seed(1)
    wp, wv = torch.randn(2, 3, A, generator=g, dtype=torch.float64), torch.randn(2, 3, generator=g, dtype=torch.float64)

    def f():
        (fp, fv, *_), _ = lr._unrolled(t)
        return torch.sum(fp * wp) + torch.sum(fv * wv)
    names = ["lstm.w", "lstm.w", "lstm.w", "lstm.b", "actor1.w", "critic1.w"]
    idx = [(10, 5), (3392 + 7, 300), (3392 + 255, 1023), (600,), (4, 9), (200, 17)]
    grads = torch.autograd.grad(f(), [lr.params[n] for n in set(names)])
    gmap = dict(zip(set(names), grads))
    eps = 1e-6
    with torch.no_grad():
        for n, i in zip(names, idx):
            p = lr.params[n]
            p[i] += eps
            up = float(f())
            p[i] -= 2 * eps
            dn = float(f())
            p[i] += eps
            fd = (up - dn) / (2 * eps)
            an = float(gmap[n][i])
            assert abs(fd - an) <= 1e-6 * max(abs(an), 1e-3), (n, i, fd, an)


@pytest.fixture(scope="module")
def rows(params):
    """Every oracle row the parity harness compares, for the correct oracle and each injected defect."""
    batch = ro.with_dones(synthetic.make_batch(4, T=T, A=A, seed=5), [(0, 0), (1, 2), (2, 3), (3, T - 1), (1, 4)])
    args = [batch[k] for k in synthetic.TRAIN_FIELDS]
    out = {}
    for bug in (None,) + ro.BUGS:
        lr = ro.RecurrentLearner(params, bug=bug, trajectory=T, num_action=A)
        o, g = lr.gradients(*args)
        r = {"act/h1": o["taps"]["h1"].detach().numpy(), "act/hin": o["taps"]["hin"].detach().numpy()}
        for k in ("pi_loss", "total_loss"):
            r["loss/" + k] = float(o[k].detach())
        for n in g:
            r["grad/" + n] = g[n].detach().numpy()
        out[bug] = r
    return out


@pytest.mark.parametrize("bug,row", [("restart_ignored", "act/hin"), ("zero_reset", "act/hin"),
                                     ("bptt_across_done", "grad/lstm.w"), ("wgrad_recorded_h", "grad/lstm.w"),
                                     ("wh_in_lstm_fwd", "act/h1")])
def test_each_defect_misses_its_row_by_10x(rows, bug, row):
    import parity
    ok = rows[None]
    worst = max(parity.rel_err(rows[bug][k], ok[k]) for k in ok if k.startswith(row))
    assert worst >= 10 * parity.TOL, (bug, row, worst)


def _config(**kw):
    from distributed_reinforcement_learning_b200 import _native as N
    cfg = N.LearnerConfig(4, 20, 84, 84, 4, 18, 256, 0.99, 6e-4, 0.0, 1e9, 1.0, 0.05, 40.0,
                          N.REWARD_CLIPPING["abs_one"], 99, 2, 1, 0, 0)
    for k, v in kw.items():
        setattr(cfg, k, v)
    return N, cfg


@pytest.mark.parametrize("value", [2, -1, 7])
def test_recurrent_field_is_validated_before_any_device_lookup(value):
    N, cfg = _config(recurrent=value)
    h = C.c_void_p()
    assert N.lib.drl_learner_create(C.byref(cfg), C.byref(h)) == N.DRL_ERR_INVALID
    assert "recurrent must be 0" in N.lib.drl_last_error().decode()


@pytest.mark.parametrize("mode", [1, 3])
def test_recurrent_refuses_math_modes_it_does_not_run(mode):
    N, cfg = _config(recurrent=1, math_mode=mode)
    h = C.c_void_p()
    assert N.lib.drl_learner_create(C.byref(cfg), C.byref(h)) == N.DRL_ERR_INVALID
    assert "math mode %d" % mode in N.lib.drl_last_error().decode()


@pytest.mark.parametrize("mode", [0, 2, 5])
def test_valid_recurrent_config_reaches_the_device_lookup(mode):
    """device 99 does not exist (with or without a GPU): a valid config fails at the device lookup, not before"""
    N, cfg = _config(recurrent=1, math_mode=mode)
    h = C.c_void_p()
    assert N.lib.drl_learner_create(C.byref(cfg), C.byref(h)) == N.DRL_ERR_CUDA
    assert "not available" in N.lib.drl_last_error().decode()


def test_agent_mode_switch_keeps_the_constructor_and_the_state(native):
    """impala.Agent keeps the reference's 14 constructor arguments; set_recurrent picks the mode of the learner engine
    it builds at the next step, and the parameters and RMSProp state stay."""
    from distributed_reinforcement_learning_b200.agent import impala
    a = impala.Agent(20, [84, 84, 4], 18, 256, 0.99, 6e-4, 0.0, 1e9, 1.0, 0.05, 40.0, "abs_one", "rec_cpu", "rec_cpu")
    a.set_session(None)
    p0 = a._params.copy()
    assert a.recurrent is False
    a.set_recurrent(True)
    assert a.recurrent is True and a._engine is None and np.array_equal(a._params, p0)
    a.set_recurrent(False)
    assert a.recurrent is False
