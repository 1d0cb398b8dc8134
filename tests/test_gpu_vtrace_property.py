"""-m gpu: hypothesis-driven property tests of the CUDA V-trace kernels against the NumPy oracle (SURVEY.md section 4):
random B in [1,64], T in [3,32], A in [2,18], done masks, extreme importance ratios, out-of-range actions (tf.one_hot
selects nothing), both stand-alone entry points (``drl_vtrace_from_importance_weights`` / ``_from_softmax``), the
committed reference-executed golden vector, and the FUSED learner kernel (V-trace x2 + pg_advantage + losses inside
``drl_learner_step``) through its taps -- fed the engine's own policy/value, so only the V-trace/loss arithmetic is
under test there.  Size-independent properties: on-policy => n-step return; all done => one-step target; linearity in
(rewards, values, bootstrap) at fixed rho; clip threshold monotonicity."""
import os

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from oracle import vtrace_np

pytestmark = pytest.mark.gpu
RTOL = 1e-4
SETTINGS = dict(max_examples=40, deadline=None, derandomize=True,
                suppress_health_check=[HealthCheck.function_scoped_fixture, HealthCheck.too_slow])


def _vt():
    from distributed_reinforcement_learning_b200.optimizer import vtrace
    return vtrace


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30)) if b.size else 0.0


def _softmax(x):
    e = np.exp(x - x.max(-1, keepdims=True))
    return (e / e.sum(-1, keepdims=True)).astype(np.float32)


@settings(**SETTINGS)
@given(B=st.integers(1, 64), T=st.integers(1, 32), seed=st.integers(0, 2 ** 31 - 1), spread=st.sampled_from([0.3, 1.0, 6.0]),
       p_done=st.sampled_from([0.0, 0.1, 0.7, 1.0]), clip=st.sampled_from([None, 0.5, 1.0, 3.0]))
def test_from_importance_weights_property(native, B, T, seed, spread, p_done, clip):
    rng = np.random.default_rng(seed)
    kw = dict(log_rhos=(rng.standard_normal((T, B)) * spread).astype(np.float32),
              discounts=((rng.random((T, B)) >= p_done) * 0.99).astype(np.float32),
              rewards=(rng.standard_normal((T, B)) * 3).astype(np.float32),
              values=rng.standard_normal((T, B)).astype(np.float32),
              bootstrap_value=rng.standard_normal(B).astype(np.float32))
    vs, rho = _vt().from_importance_weights(clip_rho_threshold=clip, **kw)
    k64 = {k: v.astype(np.float64) for k, v in kw.items()}
    evs, erho = vtrace_np.from_importance_weights(clip_rho_threshold=clip, **k64)
    assert np.all(np.isfinite(vs)) and _rel(vs, evs) < RTOL and _rel(rho, erho) < RTOL
    if clip is not None:
        assert rho.max() <= clip * (1 + 1e-6)
    if p_done == 1.0:                                   # App. C.3: vs_t = V_t + rho_t (r_t - V_t)
        exp = k64["values"] + erho * (k64["rewards"] - k64["values"])
        assert _rel(vs, exp) < RTOL
    # linearity in (rewards, values, bootstrap) at fixed log_rhos / discounts: vs(2x) == 2 vs(x)
    kw2 = dict(kw, rewards=kw["rewards"] * 2, values=kw["values"] * 2, bootstrap_value=kw["bootstrap_value"] * 2)
    vs2, _ = _vt().from_importance_weights(clip_rho_threshold=clip, **kw2)
    assert _rel(vs2, 2.0 * evs) < RTOL


@settings(**SETTINGS)
@given(B=st.integers(1, 64), T=st.integers(1, 32), A=st.integers(2, 18), seed=st.integers(0, 2 ** 31 - 1),
       sharp=st.sampled_from([0.5, 2.0, 8.0]), p_done=st.sampled_from([0.0, 0.05, 1.0]))
def test_from_softmax_property(native, B, T, A, seed, sharp, p_done):
    rng = np.random.default_rng(seed)
    mu, pi = _softmax(rng.standard_normal((B, T, A)) * sharp), _softmax(rng.standard_normal((B, T, A)) * sharp)
    mu, pi = np.maximum(mu, 1e-30).astype(np.float32), np.maximum(pi, 1e-30).astype(np.float32)
    act = rng.integers(0, A, (B, T)).astype(np.int32)
    disc = ((rng.random((B, T)) >= p_done) * 0.99).astype(np.float32)
    rew, val, nval = (rng.standard_normal((B, T)).astype(np.float32) for _ in range(3))
    vs, rho = _vt().from_softmax(mu, pi, act, disc, rew, val, nval, A)
    f = lambda x: x.astype(np.float64)
    evs, erho = vtrace_np.from_softmax(f(mu), f(pi), act, f(disc), f(rew), f(val), f(nval), A)
    ok = np.isfinite(evs)                               # sharp=8 can underflow a float32 probability to 0 -> inf/nan in both
    assert np.array_equal(np.isfinite(vs), ok)
    assert _rel(np.where(ok, vs, 0), np.where(ok, evs, 0)) < RTOL and _rel(rho, erho) < RTOL
    # on-policy, no dones (App. C.2): vs is the n-step return, whatever the values are
    if p_done == 0.0:
        vs_on, rho_on = _vt().from_softmax(pi, pi, act, disc, rew, val, nval, A)
        ret = np.zeros((B, T))
        acc = f(nval)[:, -1]
        for t in range(T - 1, -1, -1):
            acc = f(rew)[:, t] + 0.99 * acc
            ret[:, t] = acc
        assert _rel(vs_on, ret) < RTOL and np.allclose(rho_on, 1.0, atol=1e-6)


def test_out_of_range_actions_select_nothing(native):
    """tf.one_hot(a, A) with a outside [0, A) is the zero vector: log(0) - log(0) = nan in the reference; the kernels must
    neither read out of bounds nor disturb the other trajectories."""
    rng = np.random.default_rng(5)
    B, T, A = 6, 9, 7
    mu, pi = _softmax(rng.standard_normal((B, T, A))), _softmax(rng.standard_normal((B, T, A)))
    act = rng.integers(0, A, (B, T)).astype(np.int32)
    act[2, 3], act[4, 0] = A, -1
    disc = np.full((B, T), 0.99, np.float32)
    rew, val, nval = (rng.standard_normal((B, T)).astype(np.float32) for _ in range(3))
    vs, rho = _vt().from_softmax(mu, pi, act, disc, rew, val, nval, A)
    f = lambda x: x.astype(np.float64)
    with np.errstate(all="ignore"):
        evs, erho = vtrace_np.from_softmax(f(mu), f(pi), act, f(disc), f(rew), f(val), f(nval), A)
    good = [b for b in range(B) if b not in (2, 4)]
    assert _rel(vs[good], evs[good]) < RTOL and _rel(rho[good], erho[good]) < RTOL
    # The selected probability is 0 there: log(0) - log(0) = nan.  What min(1, nan) yields is unspecified in the reference
    # (Eigen's scalar min returns 1, its SSE packet min returns nan; NumPy propagates nan; CUDA's fminf returns 1), so only
    # memory safety and the isolation of the other trajectories are asserted, not the value at the poisoned step.
    assert vs.shape == evs.shape and rho.shape == erho.shape


def test_golden_reference_executed_vector_on_the_cuda_kernel(native):
    """tests/golden/vtrace_T18_B8.npz: inputs and outputs of the reference's own optimizer/vtrace.py
    from_importance_weights, executed over oracle/tf1_shim (make_golden.py) -- fed to the CUDA kernel."""
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "vtrace_T18_B8.npz"))
    assert "reference files executed" in str(z["source"])
    vs, rho = _vt().from_importance_weights(z["log_rhos"], z["discounts"], z["rewards"], z["values"], z["bootstrap_value"])
    assert _rel(vs, z["vs"]) < RTOL and _rel(rho, z["clipped_rhos"]) < RTOL


@settings(max_examples=12, deadline=None, derandomize=True,
          suppress_health_check=[HealthCheck.function_scoped_fixture, HealthCheck.too_slow])
@given(B=st.integers(1, 6), T=st.integers(3, 32), A=st.integers(2, 18), seed=st.integers(0, 10 ** 6),
       clipping=st.sampled_from(["abs_one", "soft_asymmetric"]))
def test_fused_learner_vtrace_kernel_property(native, B, T, A, seed, clipping):
    """The fused kernel of the learner step (both V-trace windows, pg_advantage, the three loss sums): its taps and
    losses against optimizer/vtrace.py (NumPy oracle, float64) evaluated on the ENGINE'S OWN policy / value outputs."""
    check_fused_learner_vtrace(B, T, A, seed, clipping)


def check_fused_learner_vtrace(B, T, A, seed, clipping):
    import parity
    from oracle import impala_torch as it
    from oracle import synthetic
    batch, params, cfg = parity.make_case(B, T, A, seed=seed, reward_clipping=clipping)
    batch["reward"] = (batch["reward"] * 3).astype(np.float32)         # exercise both clipping branches
    batch["done"] = np.random.default_rng(seed).random((B, T)) < 0.2
    eng = parity.native_learner(batch, params, cfg)
    try:
        eng.stage(0, *[batch[k] for k in synthetic.TRAIN_FIELDS])
        out = eng.step(0)
        taps = eng.taps()
        M = B * T
        pol = parity.to_batch_major(eng.read_buffer("policy", M * A).reshape(M, A), B, T).reshape(B, T, A).astype(np.float64)
        val = parity.to_batch_major(eng.read_buffer("value", M), B, T).reshape(B, T).astype(np.float64)
    finally:
        eng.close()
    r = batch["reward"].astype(np.float64)
    if clipping == "abs_one":
        cr = np.clip(r, -1.0, 1.0)
    else:
        sq = np.tanh(r / 5.0)
        cr = np.where(r < 0, 0.3 * sq, sq) * 5.0
    disc = (~batch["done"]).astype(np.float64) * 0.99
    mu = batch["behavior_policy"].astype(np.float64)
    sd = vtrace_np.split_data
    (fp, mp_, _), (fv, mv, lv) = sd(pol), sd(val)
    (fa, ma, _), (fr, mr, _), (fd, md, _), (fb, mb, _) = sd(batch["action"]), sd(cr), sd(disc), sd(mu)
    vs, rho = vtrace_np.from_softmax(fb, fp, fa, fd, fr, fv, mv, A)
    vs1, _ = vtrace_np.from_softmax(mb, mp_, ma, md, mr, mv, lv, A)
    adv = rho * (fr + fd * vs1 - fv)
    for k, e in (("vs", vs), ("clipped_rho", rho), ("vs_plus_1", vs1), ("pg_advantage", adv)):
        assert _rel(taps[k], e) < RTOL, k
    assert abs(out["pi_loss"] - vtrace_np.compute_policy_gradient_loss(fp, fa, adv, A)) <= RTOL * max(1.0, abs(out["pi_loss"]))
    assert abs(out["baseline_loss"] - vtrace_np.compute_baseline_loss(vs, fv)) <= RTOL * max(1.0, abs(out["baseline_loss"]))
    assert abs(out["entropy"] - vtrace_np.compute_entropy_loss(fp)) <= RTOL * max(1.0, abs(out["entropy"]))
