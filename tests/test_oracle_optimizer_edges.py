"""CPU self-checks of what the optimizer-edge GPU tests (tests/test_gpu_config_edges.py) compare against: the Adam
update the parity harnesses expect (``apex_parity.adam_expected``) with clipping engaged and a restored state, the
float32 polynomial learning-rate decay past and inside its schedule, and the plumbing that hands the optimizer
settings and the initial optimizer state to BOTH the CUDA learner and the oracle (checked with a stand-in for the
native learner, so no GPU is needed)."""
import numpy as np
import pytest
import torch

import a3c_parity as a3p
import apex_parity as ap
import parity
import r2d2_parity as rp
from oracle import a3c_torch as at
from oracle import apex_torch as ax
from oracle import impala_torch as it
from oracle import r2d2_torch as rt


def _flat64(tensors):
    return np.concatenate([v.detach().to(torch.float64).reshape(-1).numpy() for v in tensors.values()])


def _adam_state(n, seed):
    rng = np.random.default_rng(seed)
    return dict(m=(rng.standard_normal(n) * 1e-4).astype(np.float32), v=rng.uniform(1e-10, 1e-6, n).astype(np.float32),
                step=10 ** 6, beta1_power=float(np.float32(0.9 ** 1000)), beta2_power=float(np.float32(0.999 ** 1000)))


class _NoEngine:
    def set_opt_state(self, *a):
        pass


# ---- adam_expected against the oracles' own Adam ------------------------------------------------------------------------
@pytest.mark.parametrize("family", ["apex", "a3c"])
def test_adam_expected_equals_oracle_update_clipped_restored(family):
    """With clipping engaged (clip 0.1 < ||g||) and a mid-training Adam state, the update adam_expected predicts from the
    gradient equals the float64 update of ax.Learner / at.Learner from the same gradient."""
    A, clip = 4, 0.1
    b = ax.make_transitions(2, A=A, seed=17)
    if family == "apex":
        L = ax.Learner(ax.init_params(0, torch.float32, num_action=A), ax.init_params(1, torch.float32, num_action=A),
                       torch.float64, num_action=A, gradient_clip_norm=clip, learning_frame=2e6)
        unflat = lambda f: ax.unflatten_params(f, torch.float64, num_action=A)     # noqa: E731
        n = ax.param_count(num_action=A)
    else:
        L = at.Learner(at.init_params(0, torch.float32, num_action=A), torch.float64, num_action=A,
                       gradient_clip_norm=clip, learning_frame=2e6)
        unflat = lambda f: at.unflatten_params(f, torch.float64, num_action=A)     # noqa: E731
        n = at.param_count(num_action=A)
    st = _adam_state(n, 5)
    assert ap.load_adam_state(_NoEngine(), L, st, unflat) == 10 ** 6
    p0, m0, v0 = _flat64(L.params), _flat64(L.m), _flat64(L.v)
    b1p, b2p = float(L.beta1_power), float(L.beta2_power)
    if family == "apex":
        _, _, g, gn, lr = L.distributed_train(*[b[k] for k in ax.TRAIN_FIELDS], return_all=True)
    else:
        res, _, g, gn = L.train(*[b[k] for k in at.TRAIN_FIELDS], return_all=True)
        lr = res[3]
    assert gn > clip                                           # the clip is engaged
    assert lr == it.polynomial_decay_f32(1e-4, 10 ** 6, 2e6, 0.0) and 0 < lr < np.float32(1e-4)
    exp_p, exp_m, exp_v = ap.adam_expected(p0, _flat64(g), m0, v0, gn, clip, float(lr), b1p, b2p)
    assert parity.rel_err(_flat64(L.m), exp_m) < 1e-12
    assert parity.rel_err(_flat64(L.v), exp_v) < 1e-12
    assert np.max(np.abs(_flat64(L.params) - exp_p)) <= 1e-12 * np.max(np.abs(exp_p - p0))
    # without the clip the prediction is a different update: the case does depend on it
    _, unclipped_m, _ = ap.adam_expected(p0, _flat64(g), m0, v0, gn, 1e30, float(lr), b1p, b2p)
    assert parity.rel_err(unclipped_m, exp_m) > 0.1


# ---- polynomial decay in float32 ---------------------------------------------------------------------------------------
def test_polynomial_decay_past_the_schedule_is_end_rate():
    for step in (2, 3, 10 ** 7):
        assert it.polynomial_decay_f32(6e-4, step, 2, 1e-4) == np.float32(1e-4)
    assert it.polynomial_decay_f32(6e-4, 0, 2, 1e-4) == np.float32(np.float32(6e-4) - np.float32(1e-4)) + np.float32(1e-4)


def test_polynomial_decay_midpoint_is_tf1_float32():
    """tf.train.polynomial_decay with float32 learning rate: (lr - end) * (1 - step / decay) ** 1 + end, every operation
    rounded to float32."""
    f = np.float32
    mid = f(f(f(6e-4) - f(1e-4)) * f(f(1.0) - f(1.0) / f(2.0))) + f(1e-4)
    assert it.polynomial_decay_f32(6e-4, 1, 2, 1e-4) == mid
    assert abs(float(mid) - 3.5e-4) <= float(np.spacing(f(3.5e-4)))
    # step 1e7 of 2e7: exactly half of the start rate
    assert it.polynomial_decay_f32(6e-4, 10 ** 7, 2e7, 0.0) == f(6e-4) * f(0.5)
    # the global step is cast to float32 first: 2^24 + 1 rounds to 2^24
    assert it.polynomial_decay_f32(1.0, 2 ** 24 + 1, 2 ** 25, 0.0) == f(0.5)


# ---- the harness options reach both sides --------------------------------------------------------------------------------
class _Stop(Exception):
    pass


class _StubEngine:
    """Records what the harness gives the native learner; any other use ends the run (no GPU here)."""
    num_slots = 2

    def __init__(self, log, kw):
        self.log = log
        log["kw"] = kw

    def set_opt_state(self, *a):
        self.log["opt_state"] = a

    def close(self):
        self.log["closed"] = True

    def __getattr__(self, name):
        raise _Stop(name)


def _record_oracle(monkeypatch, module, log):
    base = module.Learner

    class Rec(base):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            log["oracle"] = self
    monkeypatch.setattr(module, "Learner", Rec)


def test_impala_harness_passes_options_to_both(monkeypatch):
    log = {}
    _record_oracle(monkeypatch, it, log)
    monkeypatch.setattr(parity, "native_learner", lambda batch, params, cfg, **kw: _StubEngine(log, kw))
    opt = dict(gradient_clip_norm=1.0, start_learning_rate=6e-4, end_learning_rate=1e-4, learning_frame=2e7)
    ms = np.random.default_rng(0).uniform(0.05, 2.0, it.param_count(num_action=6)).astype(np.float32)
    with pytest.raises(_Stop):
        parity.compare_step(2, T=5, A=6, opt=opt, init_state=dict(ms=ms, step=10 ** 7), math_mode=1)
    assert log["kw"] == dict(opt, math_mode=1) and log["closed"]
    L = log["oracle"]
    assert all(L.cfg[k] == v for k, v in opt.items())
    assert log["opt_state"][0] is ms and log["opt_state"][1] == 10 ** 7
    assert L.step == 10 ** 7 and np.array_equal(_flat64(L.ms), ms.astype(np.float64))
    # defaults: nothing extra reaches the native learner, and the oracle keeps its defaults and fresh slots
    log.clear()
    with pytest.raises(_Stop):
        parity.compare_step(2, T=5, A=6)
    assert log["kw"] == {} and "opt_state" not in log
    assert all(log["oracle"].cfg[k] == it.DEFAULT_CFG[k] for k in parity.OPT_KEYS)
    assert log["oracle"].step == 0 and all(bool((v == 1).all()) for v in log["oracle"].ms.values())
    with pytest.raises(ValueError):
        parity.compare_step(2, T=5, A=6, opt=dict(learning_rate=1e-3))


@pytest.mark.parametrize("family", ["apex", "a3c"])
def test_adam_harnesses_pass_options_to_both(monkeypatch, family):
    log = {}
    if family == "apex":
        oracle, compare = ax, ap.compare_step
        monkeypatch.setattr(ap, "native_apex", lambda B, A, params, target, **kw: _StubEngine(log, kw))
    else:
        oracle, compare = at, a3p.compare_step
        monkeypatch.setattr(a3p, "native_a3c", lambda B, A, params, **kw: _StubEngine(log, kw))
    _record_oracle(monkeypatch, oracle, log)
    opt = dict(gradient_clip_norm=0.5, start_learning_rate=6e-4, end_learning_rate=1e-4, learning_frame=2)
    st = _adam_state(oracle.param_count(num_action=4), 1)
    with pytest.raises(_Stop):
        compare(2, A=4, opt=opt, init_state=st)
    assert log["kw"] == dict(opt, reward_clipping="abs_one") and log["closed"]
    L = log["oracle"]
    assert all(L.cfg[k] == v for k, v in opt.items())
    assert log["opt_state"] == (st["m"], st["v"], st["step"], st["beta1_power"], st["beta2_power"])
    assert L.step == st["step"] and L.beta1_power == np.float32(st["beta1_power"])
    assert L.beta2_power == np.float32(st["beta2_power"])
    assert np.array_equal(_flat64(L.m), st["m"].astype(np.float64))
    assert np.array_equal(_flat64(L.v), st["v"].astype(np.float64))
    log.clear()
    with pytest.raises(_Stop):
        compare(2, A=4)
    assert log["kw"] == dict(reward_clipping="abs_one") and "opt_state" not in log
    assert all(log["oracle"].cfg[k] == oracle.DEFAULT_CFG[k] for k in ap.OPT_KEYS)
    assert log["oracle"].step == 0 and log["oracle"].beta1_power == np.float32(0.9)


def test_r2d2_harness_passes_options_to_both(monkeypatch):
    log = {}
    _record_oracle(monkeypatch, rt, log)
    monkeypatch.setattr(rp, "native_r2d2", lambda B, S, bi, A, C, params, target, **kw: _StubEngine(log, kw))
    st = _adam_state(rt.param_count(num_action=4, lstm_size=64, input_shape=(84, 84, 1)), 2)
    with pytest.raises(_Stop):
        rp.compare_step(2, S=6, bi=2, opt=dict(learning_rate=3e-4), init_state=st)
    assert log["kw"] == dict(learning_rate=3e-4)
    L = log["oracle"]
    assert L.cfg["learning_rate"] == 3e-4 and L.step == st["step"]
    assert np.array_equal(_flat64(L.v), st["v"].astype(np.float64))
    log.clear()
    with pytest.raises(_Stop):
        rp.compare_step(2, S=6, bi=2)
    assert log["kw"] == {} and log["oracle"].cfg["learning_rate"] == rt.LR
    with pytest.raises(ValueError):
        rp.compare_step(2, S=6, bi=2, opt=dict(gradient_clip_norm=1.0))    # R2D2 does not clip


def test_r2d2_oracle_learning_rate_setting():
    """rt.Learner's Adam rate is the ``learning_rate`` setting (default agent/r2d2.py's 1e-4)."""
    kwp = dict(num_action=4, lstm_size=64, input_shape=(84, 84, 1))
    b = rt.make_sequences(1, S=4, seed=3)
    ups = []
    for lr in (None, 1e-4, 3e-4):
        cfg = {} if lr is None else dict(learning_rate=lr)
        L = rt.Learner(rt.init_params(0, torch.float32, **kwp), rt.init_params(1, torch.float32, **kwp), torch.float64,
                       seq_len=4, burn_in=1, **kwp, **cfg)
        p0 = _flat64(L.params)
        L.train(*[b[k] for k in rt.TRAIN_FIELDS])
        ups.append(_flat64(L.params) - p0)
    assert np.array_equal(ups[0], ups[1])
    assert np.allclose(ups[2], ups[1] * float(np.float32(3e-4)) / float(np.float32(1e-4)), rtol=1e-9, atol=0)


def test_r2d2_done_overrides():
    base = rt.make_sequences(3, S=20, A=4, input_shape=(84, 84, 1), seed=5)
    same = rp.make_batch(3, 20, 4, 1, 5)
    assert all(np.array_equal(base[k], same[k]) for k in base)
    b = rp.make_batch(3, 20, 4, 1, 5, done_rate=0.5, done_ends=True)
    assert b["done"][:, 0].all() and b["done"][:, -1].all() and 0.4 < b["done"].mean() < 0.8
    assert all(np.array_equal(base[k], b[k]) for k in base if k != "done")
