"""CPU checks of tests/optimizer_parity.py, the float64 references of the optimizer tails:

* fed one gradient, they reproduce the oracles' own RMSProp (impala_torch) and Adam updates (apex_torch, a3c_torch,
  apex_parity.adam_expected);
* their bounds are sharp: each mutation of the update a kernel could plausibly carry exceeds the bound at least 10x on
  some element of the same inputs;
* a NaN or infinite global norm poisons every parameter in the oracles, as tf.clip_by_global_norm does in TF 1.14."""
import numpy as np
import pytest
import torch

import apex_parity as ap
import optimizer_parity as op
import parity
from oracle import a3c_torch as at
from oracle import apex_torch as ax
from oracle import impala_torch as it

f32 = np.float32
GS = 0.5                       # a data-parallel grad_scale of the mutation cases


def _gradient(n, seed, big=1.0):
    """A gradient with magnitudes spread over 1e-9 .. big (the small elements are where epsilon placement shows)."""
    rng = np.random.default_rng(seed)
    g = rng.standard_normal(n) * 10.0 ** rng.uniform(-9, 0, n) * big
    return g.astype(np.float32)


def _fed(L, g_named, extra):
    """Make the oracle learner's next step see exactly the gradient ``g_named``: its loss becomes sum(p * g)."""
    def losses(*a, **k):
        loss = sum((p * g_named[n].to(p.dtype)).sum() for n, p in L.params.items())
        return dict(extra, total_loss=loss, value_loss=loss, taps={})
    L.losses = losses


def _named(flat, unflatten, **kw):
    return unflatten(np.asarray(flat, np.float32), torch.float64, **kw)


def _flat64(d):
    return np.concatenate([v.detach().double().reshape(-1).numpy() for v in d.values()])


# ---- the references reproduce the oracles ----------------------------------------------------------------------------
@pytest.mark.parametrize("clip", [40.0, 1e-3])
def test_rmsprop_reference_matches_impala_oracle(clip):
    L = it.Learner(dtype=torch.float64, num_action=6, gradient_clip_norm=clip, start_learning_rate=6e-4,
                   end_learning_rate=1e-4, learning_frame=1000)
    L.step = 7
    p0 = f32(it.flatten_params(L.params))
    L.params = type(L.params)((k, v.detach().float().double().requires_grad_(True)) for k, v in L.params.items())
    g = _gradient(p0.size, 1, big=0.01)
    gn = _named(g, it.unflatten_params, num_action=6)
    z = torch.zeros((), dtype=torch.float64)
    _fed(L, gn, dict(pi_loss=z, baseline_loss=z, entropy=z))
    _, _, _, gnorm = L.train(*[None] * 8, return_all=True)
    kind, norm, _ = op.global_norm(g, g.size)
    assert kind == "finite" and abs(norm - gnorm) <= 1e-12 * norm
    assert (norm > clip) == (clip < 1)
    lr = op.learning_rate(6e-4, 1e-4, 1000, 7)
    ref, _ = op.rmsprop(p0, np.ones_like(p0), g, op.clip_scale(f32(norm), clip), lr)
    assert parity.rel_err(ref["w"] - p0, _flat64(L.params) - p0) < parity.TOL
    assert parity.rel_err(ref["ms"], _flat64(L.ms)) < parity.TOL


@pytest.mark.parametrize("family", ["apex", "a3c"])
@pytest.mark.parametrize("clip", [40.0, 1e-3])
def test_adam_reference_matches_apex_and_a3c_oracles(family, clip):
    mod = ax if family == "apex" else at
    cfg = dict(num_action=4, gradient_clip_norm=clip, start_learning_rate=1e-4, end_learning_rate=3e-5, learning_frame=1000)
    L = mod.Learner(dtype=torch.float64, **cfg)
    p0 = f32(ax.flatten_params(L.params))
    L.params = type(L.params)((k, v.detach().float().double().requires_grad_(True)) for k, v in L.params.items())
    rng = np.random.default_rng(2)
    m0 = (rng.standard_normal(p0.size) * 1e-3).astype(np.float32)
    v0 = (rng.random(p0.size) * 1e-6).astype(np.float32)
    with torch.no_grad():
        for n, t in mod.unflatten_params(m0, torch.float64, num_action=4).items():
            L.m[n].copy_(t)
        for n, t in mod.unflatten_params(v0, torch.float64, num_action=4).items():
            L.v[n].copy_(t)
    L.step, L.beta1_power, L.beta2_power = 11, f32(0.9 ** 12), f32(0.999 ** 12)
    g = _gradient(p0.size, 3, big=0.01)
    gn = _named(g, mod.unflatten_params, num_action=4)
    z = torch.zeros((), dtype=torch.float64)
    zb = torch.zeros(2, dtype=torch.float64)
    _fed(L, gn, dict(pi_loss=z, baseline_loss=z, entropy=z, target_value=zb, state_action_value=zb))
    if family == "apex":
        L.distributed_train(*[None] * 6, is_weight=None)
    else:
        L.train(*[None] * 6)
    kind, norm, _ = op.global_norm(g, g.size)
    assert kind == "finite" and (norm > clip) == (clip < 1)
    lr = op.learning_rate(1e-4, 3e-5, 1000, 11)
    alpha, b1, b2 = op.adam_scalars(lr, f32(0.9 ** 12), f32(0.999 ** 12))
    assert (b1, b2) == (L.beta1_power, L.beta2_power)
    ref, _ = op.adam(p0, m0, v0, g, op.clip_scale(f32(norm), clip), alpha)
    assert parity.rel_err(ref["w"] - p0, _flat64(L.params) - p0) < parity.TOL
    assert parity.rel_err(ref["m"], _flat64(L.m)) < parity.TOL and parity.rel_err(ref["v"], _flat64(L.v)) < parity.TOL
    exp = ap.adam_expected(p0.astype(np.float64), g.astype(np.float64), m0.astype(np.float64), v0.astype(np.float64),
                           norm, clip, float(lr), float(f32(0.9 ** 12)), float(f32(0.999 ** 12)))
    for e, k in zip(exp, ("w", "m", "v")):
        base = p0 if k == "w" else 0.0
        assert parity.rel_err(ref[k] - base, e - base) < parity.TOL, k


# ---- the bounds are sharp -----------------------------------------------------------------------------------------------
def _case(n=20000, seed=5):
    """Inputs of the mutation cases: a padded bucket with one nonzero padding element, random slots, step 10 of a
    1000-step decay (the rates of steps 10 and 11 differ by 0.1 %), clipping engaged."""
    rng = np.random.default_rng(seed)
    g = _gradient(n, seed, big=10.0)
    idx = np.sort(rng.choice(n + 64, n, replace=False))
    bucket = np.zeros(n + 64, np.float32)
    bucket[idx] = g
    pad = op.padding_of(idx, n + 64)
    bucket[pad[3]] = 50.0
    w = rng.standard_normal(n).astype(np.float32) * 0.05
    ms = (rng.random(n) * 1e-2).astype(np.float32)
    m = (rng.standard_normal(n) * 1e-3).astype(np.float32)
    v = (rng.random(n) * 1e-6).astype(np.float32)
    v[:50] = 0.0
    m[:50] = 0.0
    return dict(g=g, bucket=bucket, idx=idx, w=w, ms=ms, m=m, v=v, clip=1.0, step=10, frame=1000, start=1e-3, end=1e-4)


def _sharp(mut, ref, bound):
    with np.errstate(all="ignore"):
        return float(np.nanmax(np.abs(mut - ref) / bound))


def _rms_mutant(c, scale, lr, decay=0.99, eps_outside=False):
    w, ms, g = [c[k].astype(np.float64) for k in ("w", "ms", "g")]
    gg = g * float(scale)
    m1 = ms + (gg * gg - ms) * float(f32(1) - f32(decay))          # TF's float32 constants
    eps = float(op.RMS_EPS)
    if eps_outside:
        return w - float(lr) * gg / (np.sqrt(m1) + eps), m1
    return w - float(lr) * gg / np.sqrt(m1 + eps), m1


def _adam_mutant(c, scale, alpha, eps_inside=False):
    w, m, v, g = [c[k].astype(np.float64) for k in ("w", "m", "v", "g")]
    gg = g * float(scale)
    m1 = m + (gg - m) * float(op.ADAM_C1)
    v1 = v + (gg * gg - v) * float(op.ADAM_C2)
    eps = float(op.ADAM_EPS)
    den = np.sqrt(v1 + eps) if eps_inside else np.sqrt(v1) + eps
    return w - m1 * float(alpha) / den, m1, v1


def test_rmsprop_bounds_reject_mutations():
    c = _case()
    npad = c["bucket"].size
    kind, norm, _ = op.global_norm(c["bucket"][c["idx"]], npad)
    assert kind == "finite" and norm > c["clip"]
    lr = op.learning_rate(c["start"], c["end"], c["frame"], c["step"])
    scale = op.clip_scale(f32(norm), c["clip"])
    ref, bd = op.rmsprop(c["w"], c["ms"], c["g"], scale, lr)
    w0, m0 = _rms_mutant(c, scale, lr)
    assert _sharp(w0, ref["w"], bd["w"]) < 1 and _sharp(m0, ref["ms"], bd["ms"]) < 1       # the mutant harness is right
    lr1 = op.learning_rate(c["start"], c["end"], c["frame"], c["step"] + 1)
    pad_norm = float(np.sqrt(np.sum(c["bucket"].astype(np.float64) ** 2)))
    mutants = {
        "epsilon outside the square root": _rms_mutant(c, scale, lr, eps_outside=True)[0],
        "decay 0.9": _rms_mutant(c, scale, lr, decay=0.9)[0],
        "clip scale omitted": _rms_mutant(c, 1.0, lr)[0],
        "learning rate of step + 1": _rms_mutant(c, scale, lr1)[0],
        "norm counts the padding": _rms_mutant(c, op.clip_scale(f32(pad_norm), c["clip"]), lr)[0],
    }
    for name, wm in mutants.items():
        assert _sharp(wm, ref["w"], bd["w"]) >= 10, name
    assert _sharp(_rms_mutant(c, scale, lr, decay=0.9)[1], ref["ms"], bd["ms"]) >= 10


def test_adam_bounds_reject_mutations():
    c = _case(seed=6)
    npad = c["bucket"].size
    kind, norm, _ = op.global_norm(c["bucket"][c["idx"]], npad, GS)
    assert kind == "finite" and norm > c["clip"]
    lr = op.learning_rate(c["start"], c["end"], c["frame"], c["step"])
    b1p, b2p = f32(0.9 ** 11), f32(0.999 ** 11)
    alpha, b1n, b2n = op.adam_scalars(lr, b1p, b2p)
    scale = op.clip_scale(f32(norm), c["clip"], GS)
    ref, bd = op.adam(c["w"], c["m"], c["v"], c["g"], scale, alpha)

    def worst(mut):
        return max(_sharp(x, ref[k], bd[k]) for x, k in zip(mut, ("w", "m", "v")))
    assert worst(_adam_mutant(c, scale, alpha)) < 1
    lr1 = op.learning_rate(c["start"], c["end"], c["frame"], c["step"] + 1)
    pad_norm = float(np.sqrt(np.sum(c["bucket"].astype(np.float64) ** 2))) * GS
    raw_norm = norm / GS
    mutants = {
        "sqrt(v + eps)": _adam_mutant(c, scale, alpha, eps_inside=True),
        "clip scale omitted": _adam_mutant(c, f32(GS), alpha),
        "learning rate of step + 1": _adam_mutant(c, scale, op.adam_scalars(lr1, b1p, b2p)[0]),
        "beta powers advanced before alpha": _adam_mutant(c, scale, op.adam_scalars(lr, b1n, b2n)[0]),
        "norm counts the padding": _adam_mutant(c, op.clip_scale(f32(pad_norm), c["clip"], GS), alpha),
        "grad_scale missing from the norm": _adam_mutant(c, op.clip_scale(f32(raw_norm), c["clip"], GS), alpha),
        "grad_scale missing from the scale": _adam_mutant(c, op.clip_scale(f32(norm), c["clip"]), alpha),
    }
    for name, mut in mutants.items():
        assert worst(mut) >= 10, name


def test_norm_bound_rejects_counted_padding_and_missing_grad_scale():
    c = _case(seed=7)
    npad = c["bucket"].size
    kind, norm, bound = op.global_norm(c["bucket"][c["idx"]], npad, GS)
    assert kind == "finite"
    pad_norm = float(np.sqrt(np.sum(c["bucket"].astype(np.float64) ** 2))) * GS
    assert abs(pad_norm - norm) >= 10 * bound
    assert abs(norm / GS - norm) >= 10 * bound
    assert op.norm_ratio(f32(norm), c["bucket"][c["idx"]], npad, GS) < 1


def test_scalars_follow_tf_float32():
    assert op.RMS_C == f32(1) - f32(0.99) and float(op.RMS_C) != 0.01
    assert op.learning_rate(1e-4, 3e-5, 1000, 2) == it.polynomial_decay_f32(1e-4, 2, 1000, 3e-5)
    alpha, b1, b2 = op.adam_scalars(f32(1e-4), f32(0.9), f32(0.999))
    assert alpha == f32(f32(f32(1e-4) * np.sqrt(f32(1) - f32(0.999))) / (f32(1) - f32(0.9)))
    assert (b1, b2) == (f32(f32(0.9) * f32(0.9)), f32(f32(0.999) * f32(0.999)))
    assert op.clip_scale(f32(0), 40.0) == f32(f32(40) * (f32(1) / f32(40)))
    assert np.isnan(op.clip_scale(f32("nan"), 40.0)) and np.isnan(op.clip_scale(f32("inf"), 40.0, 0.5))
    assert op.clip_scale(f32("nan"), 0.0, 0.5) == f32(0.5)                 # no clipping: the norm is only reported
    big = np.full(4, 1.5e19, np.float32)
    assert op.global_norm(big, 4)[0] == "inf" and op.global_norm(big[:1], 4)[0] == "finite"


# ---- non-finite norms poison every parameter, as in TF 1.14 ----------------------------------------------------------
@pytest.mark.parametrize("bad", ["nan", "inf", "overflow"])
@pytest.mark.parametrize("family", ["impala", "apex", "a3c"])
def test_oracles_make_every_parameter_nan_for_a_non_finite_norm(family, bad):
    mod = {"impala": it, "apex": ax, "a3c": at}[family]
    L = mod.Learner(dtype=torch.float32, num_action=4)
    p0 = mod.flatten_params(L.params)
    g = np.zeros(p0.size, np.float32)
    g[1::97] = 1e-3
    if bad == "overflow":
        g[:3] = 1.5e19                               # every square is finite, their float32 sum is not
    else:
        g[5] = float(bad)
    gn = mod.unflatten_params(g, torch.float32, num_action=4)
    z = torch.zeros(())
    _fed(L, gn, dict(pi_loss=z, baseline_loss=z, entropy=z, target_value=torch.zeros(2), state_action_value=torch.zeros(2)))
    with np.errstate(all="ignore"):
        if family == "impala":
            L.train(*[None] * 8)
        elif family == "apex":
            L.distributed_train(*[None] * 6, is_weight=None)
        else:
            L.train(*[None] * 6)
    assert np.isnan(mod.flatten_params(L.params)).all()
    assert op.global_norm(g, g.size)[0] == ("nan" if bad == "nan" else "inf")


def test_oracle_scale_of_a_zero_norm_is_one():
    assert it.clip_scale(0.0, 40.0) == 1.0 and it.clip_scale(80.0, 40.0) == 0.5 and it.clip_scale(20.0, 40.0) == 1.0
    assert np.isnan(it.clip_scale(float("nan"), 40.0)) and np.isnan(it.clip_scale(float("inf"), 40.0))
