"""-m gpu: the optimizer tails of the four learners -- ``sqnorm_partial_kernel`` + ``rmsprop_apply_kernel`` (IMPALA) and
``adam_prepare_kernel`` + ``adam_apply_kernel`` (Ape-X, A3C, R2D2) -- against the float64 references of
tests/optimizer_parity.py, element by element and scalar by scalar.

Each case drives the data-parallel halves of a learner on one GPU: (forward_backward), the gradient bucket written
through its torch view on the learner's stream, ``apply`` (with ``grad_scale`` for the Adam families), ``wait``.  The
inputs are read back before the apply (parameters, slots, step, beta powers), the outputs after it.  Every case asserts
the edge it claims (the norm above the clip, subnormal squares present, an infinite norm, a step that float32 rounds)."""
import ctypes as C

import numpy as np
import pytest
import torch

import optimizer_parity as op
import parity
from oracle import a3c_torch as at
from oracle import apex_torch as ax
from oracle import r2d2_torch as rt
from oracle import synthetic

pytestmark = pytest.mark.gpu

f32 = np.float32
FRAME = 2 ** 24 + 3                                  # learning_frame: a step of 2^24 + 1 rounds in float32
SCHED = dict(start_learning_rate=6e-4, end_learning_rate=1e-4, learning_frame=FRAME)
R2D2_LR = 1e-4
CLIP_ON = 1e-3                                       # below every real gradient norm here
ADAM = ("apex", "a3c", "r2d2")
WORST = {}


# ---- learners -----------------------------------------------------------------------------------------------------------
def _make(fam, clip, B=None, A=None, **kw):
    """-> (engine, stage()) at the benchmark shapes unless B is given."""
    if fam == "impala":
        B = B or 32
        batch, params, cfg = parity.make_case(B, 20 if B >= 32 else 5, A or 18, seed=11)
        eng = parity.native_learner(batch, params, cfg, gradient_clip_norm=clip, **SCHED, **kw)
        return eng, lambda: eng.stage(0, *[batch[k] for k in synthetic.TRAIN_FIELDS])
    A = A or 4
    if fam == "r2d2":
        from distributed_reinforcement_learning_b200.r2d2_learner import NativeR2D2Learner
        B = B or 16
        S, BI = (80, 40) if B >= 16 else (6, 2)
        kwp = dict(num_action=A, lstm_size=64, input_shape=(84, 84, 1))
        eng = NativeR2D2Learner(batch=B, seq_len=S, burn_in=BI, num_action=A, learning_rate=R2D2_LR, **kw)
        eng.set_params(rt.flatten_params(rt.init_params(0, torch.float32, **kwp)), 0)
        eng.set_params(rt.flatten_params(rt.init_params(1, torch.float32, **kwp)), 1)
        b = rt.make_sequences(B, S=S, A=A, seed=12)
        return eng, lambda: eng.stage(0, b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0],
                                      b["reward"], b["done"], b["weight"])
    B = B or 32
    batch = ax.make_transitions(B, A=A, seed=13)
    pm = ax.flatten_params(ax.init_params(0, torch.float32, num_action=A))
    if fam == "apex":
        from distributed_reinforcement_learning_b200.apex_learner import NativeApexLearner
        eng = NativeApexLearner(batch=B, num_action=A, gradient_clip_norm=clip, **SCHED, **kw)
        eng.set_params(pm, 0)
        eng.set_params(ax.flatten_params(ax.init_params(1, torch.float32, num_action=A)), 1)
    else:
        from distributed_reinforcement_learning_b200.a3c_learner import NativeA3CLearner
        eng = NativeA3CLearner(batch=B, num_action=A, gradient_clip_norm=clip, **SCHED, **kw)
        eng.set_params(pm)
    fields = ax.TRAIN_FIELDS if fam == "apex" else at.TRAIN_FIELDS
    return eng, lambda: eng.stage(0, *[batch[k] for k in fields])


_CACHE = {}


def _learner(fam, clip):
    """One learner per family and clip, reused across cases, with its packed <-> padded index map."""
    key = (fam, clip)
    if key not in _CACHE:
        eng, stage = _make(fam, clip)
        idx, npad = op.bucket_index_map(eng)
        _CACHE[key] = (eng, stage, idx, npad)
    return _CACHE[key]


@pytest.fixture(scope="module", autouse=True)
def _close_learners():
    yield
    for eng, *_ in _CACHE.values():
        eng.close()
    _CACHE.clear()
    if WORST:
        print("\nworst |gpu - ref| / bound per family and tensor:")
        for k in sorted(WORST):
            print("  %-8s %-6s %.3g" % (k[0], k[1], WORST[k]))


# ---- state ------------------------------------------------------------------------------------------------------------
def _state(fam, n, kind, seed=3):
    """Optimizer state -> dict(step, slots..., b1p, b2p)."""
    rng = np.random.default_rng(seed)
    step = {"fresh": 0, "restored": 333, "rounding_step": 2 ** 24 + 1, "end_rate": 2 ** 24 + 5,
            "subnormal_powers": 50, "zero_powers": 50}[kind]
    fresh = kind == "fresh"
    if fam == "impala":
        ms = np.ones(n, np.float32) if fresh else (rng.random(n) * 1e-2).astype(np.float32)
        return dict(step=step, ms=ms)
    m = np.zeros(n, np.float32) if fresh else (rng.standard_normal(n) * 1e-3).astype(np.float32)
    v = np.zeros(n, np.float32) if fresh else (rng.random(n) * 1e-6).astype(np.float32)
    b1p, b2p = f32(0.9), f32(0.999)
    if kind == "restored":
        b1p, b2p = f32(0.9 ** 334), f32(0.999 ** 334)
    elif kind == "subnormal_powers":
        b1p = b2p = f32(np.float32(2.0 ** -149))
    elif kind == "zero_powers":
        b1p = b2p = f32(0)
    return dict(step=step, m=m, v=v, b1p=b1p, b2p=b2p)


def _load(fam, eng, w, st):
    eng.set_params(w) if fam in ("impala", "a3c") else eng.set_params(w, 0)
    if fam == "impala":
        eng.set_opt_state(st["ms"], st["step"])
    else:
        eng.set_opt_state(st["m"], st["v"], st["step"], st["b1p"], st["b2p"])


def _read(fam, eng):
    w = eng.get_params() if fam in ("impala", "a3c") else eng.get_params(0)
    if fam == "impala":
        ms, step = eng.get_opt_state()
        return dict(w=w, ms=ms, step=step)
    s = eng.get_opt_state()
    return dict(w=w, m=s["m"], v=s["v"], step=s["step"], b1p=f32(s["beta1_power"]), b2p=f32(s["beta2_power"]))


# ---- buckets ----------------------------------------------------------------------------------------------------------
TAIL = np.array([1.25, -0.375, 2.5, 0.0], np.float32)


def _crafted(kind, n, clip, seed=4):
    rng = np.random.default_rng(seed)
    g = np.zeros(n, np.float32)
    if kind == "one_at_clip":
        g[n // 3] = clip
    elif kind == "spread":
        g = (rng.choice([-1, 1], n) * 10.0 ** rng.uniform(-30, 3, n)).astype(np.float32)
    elif kind == "overflow":
        g = (rng.standard_normal(n) * 1e-3).astype(np.float32)
        g[[5, n // 2, n - 7]] = 1.5e19
    elif kind in ("nan", "inf"):
        g = (rng.standard_normal(n) * 1e-3).astype(np.float32)
        g[n // 5] = float(kind)
    elif kind == "random":
        g = (rng.standard_normal(n) * 10.0 ** rng.uniform(-9, 0, n) * 1e-2).astype(np.float32)
    return g


def _assert_edge(kind, g, npad, clip, gs, row_norm):
    with np.errstate(over="ignore", under="ignore"):
        g2 = g.astype(np.float32) ** 2
    if kind == "one_at_clip" and gs == 1:
        assert row_norm == f32(clip)
    if kind == "spread":
        assert ((g2 > 0) & (g2 < np.finfo(np.float32).tiny)).any() and ((g2 == 0) & (g != 0)).any()
    if kind in ("overflow", "inf"):
        assert op.global_norm(g, npad, gs)[0] == "inf" and row_norm == np.inf
        if kind == "overflow":
            assert np.isfinite(g2).all()
    if kind == "nan":
        assert np.isnan(row_norm)


def _write_bucket(eng, padded):
    b = eng._dp._tensor()
    with torch.cuda.stream(eng._dp._stream):
        b.copy_(torch.from_numpy(padded).to(b.device))
    eng._dp._stream.synchronize()


def _bucket(eng):
    eng._dp._stream.synchronize()
    return eng._dp._tensor().cpu().numpy().copy()


def _apply(fam, eng, gs):
    from distributed_reinforcement_learning_b200 import _native as N
    if fam == "impala":
        eng.apply()
    else:
        N.check(eng._fn("apply")(eng._h, C.c_float(gs)))
    out = eng.wait()
    return out[0] if isinstance(out, tuple) else out


# ---- one checked update -------------------------------------------------------------------------------------------------
def _check(fam, eng, idx, npad, clip, padded, gs, label, expect_lr=None):
    """Apply the update to the bucket ``padded`` (already written) and compare everything with the reference."""
    g, tail = padded[idx], padded[npad:npad + 4]
    st = _read(fam, eng)
    row = _apply(fam, eng, gs)
    after = _read(fam, eng)
    norm = f32(row["grad_norm"])
    assert op.norm_ratio(norm, g, npad, gs if fam != "impala" else 1.0) < 1, (label, norm)
    assert row["step"] == st["step"] + 1 and after["step"] == st["step"] + 1
    if fam == "r2d2":
        lr = f32(R2D2_LR)
    else:
        lr = op.learning_rate(SCHED["start_learning_rate"], SCHED["end_learning_rate"], FRAME, st["step"])
        assert f32(row["learning_rate"]) == lr, (label, row["learning_rate"], lr)
        if expect_lr is not None:
            assert lr == f32(expect_lr)
    scale = op.clip_scale(norm, clip if fam != "r2d2" else 0.0, gs)
    if fam == "impala":
        assert (row["pi_loss"], row["baseline_loss"], row["entropy"]) == tuple(float(x) for x in tail[:3])
        tot = float(tail[0]) + float(tail[1]) * 1.0 + float(tail[2]) * float(f32(0.05))
        assert abs(row["total_loss"] - tot) <= 2 * op.U * (abs(tot) + abs(float(tail[0])) + abs(float(tail[1]))) + 1e-45
        ref, bd = op.rmsprop(st["w"], st["ms"], g, scale, lr)
    else:
        names = {"apex": ("loss",), "r2d2": ("loss",), "a3c": ("pi_loss", "baseline_loss", "entropy")}[fam]
        for k, t in zip(names, tail):
            assert f32(row[k]) == f32(t * f32(gs)), (label, k)
        alpha, b1, b2 = op.adam_scalars(lr, st["b1p"], st["b2p"])
        assert (after["b1p"], after["b2p"]) == (b1, b2), label
        ref, bd = op.adam(st["w"], st["m"], st["v"], g, scale, alpha)
    for k in ref:
        r, i = op.ratio(after[k], ref[k], bd[k])
        WORST[(fam, k)] = max(WORST.get((fam, k), 0.0), r)
        assert r < 1, (label, k, r, i, float(after[k][i]), float(ref[k][i]), float(bd[k][i]))
    return row


def _full(g, npad, idx, tail=TAIL):
    padded = np.zeros(npad + 4, np.float32)
    padded[idx] = g
    padded[npad:] = tail
    return padded


# ---- real buckets -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fam,clip", [("impala", 1e30), ("impala", CLIP_ON), ("apex", 0.0), ("apex", CLIP_ON),
                                      ("a3c", 0.0), ("a3c", CLIP_ON), ("r2d2", 0.0)])
def test_real_bucket_at_benchmark_shape(native, fam, clip):
    from distributed_reinforcement_learning_b200 import _native as N
    eng, stage, idx, npad = _learner(fam, clip)
    w0 = eng.get_params() if fam in ("impala", "a3c") else eng.get_params(0)
    _load(fam, eng, w0, _state(fam, idx.size, "restored"))
    stage()
    N.check(eng._fn("forward_backward")(eng._h, 0))
    padded = _bucket(eng)
    assert not padded[op.padding_of(idx, npad)].any()
    row = _check(fam, eng, idx, npad, clip, padded, 1.0, "real")
    if clip == CLIP_ON:
        assert row["grad_norm"] > clip
    elif fam == "impala":
        assert row["grad_norm"] < clip


@pytest.mark.parametrize("fam", ["impala", "apex", "a3c", "r2d2"])
@pytest.mark.parametrize("A", [2, 6, 18, 32])
def test_bucket_padding_is_zero(native, fam, A):
    """The logits / value biases are padded to a multiple of 4: after a real backward every padding element of the
    bucket is exactly 0, so the norm covers exactly the model's gradient."""
    from distributed_reinforcement_learning_b200 import _native as N
    eng, stage = _make(fam, 1.0, B=2, A=A)
    try:
        idx, npad = op.bucket_index_map(eng)
        stage()
        N.check(eng._fn("forward_backward")(eng._h, 0))
        padded = _bucket(eng)
        pad = op.padding_of(idx, npad)
        assert pad.size > 0 or npad == idx.size
        assert not padded[pad].any() and np.abs(padded[idx]).max() > 0
    finally:
        eng.close()


# ---- crafted buckets x optimizer states ---------------------------------------------------------------------------------
CRAFTED = ["zeros", "one_at_clip", "spread", "overflow", "nan", "inf"]


@pytest.mark.parametrize("fam", ["impala", "apex", "a3c", "r2d2"])
@pytest.mark.parametrize("kind", CRAFTED)
@pytest.mark.parametrize("state", ["fresh", "restored"])
def test_crafted_bucket(native, fam, kind, state):
    clip = 0.0 if fam == "r2d2" else CLIP_ON
    eng, _, idx, npad = _learner(fam, clip)
    w0 = np.random.default_rng(9).standard_normal(idx.size).astype(np.float32) * 0.05
    _load(fam, eng, w0, _state(fam, idx.size, state))
    g = _crafted(kind, idx.size, CLIP_ON)
    _write_bucket(eng, _full(g, npad, idx))
    row = _check(fam, eng, idx, npad, clip, _full(g, npad, idx), 1.0, "%s/%s" % (kind, state))
    _assert_edge(kind, g, npad, CLIP_ON, 1.0, f32(row["grad_norm"]))
    if kind in ("nan", "inf", "overflow") and fam != "r2d2":      # TF 1.14: a non-finite norm poisons every parameter
        assert np.isnan(_read(fam, eng)["w"]).all()


@pytest.mark.parametrize("fam", ["impala", "apex", "a3c", "r2d2"])
@pytest.mark.parametrize("state", ["rounding_step", "end_rate", "subnormal_powers", "zero_powers"])
def test_optimizer_state_edges(native, fam, state):
    if fam == "impala" and state.endswith("powers"):
        pytest.skip("RMSProp has no beta powers")
    clip = 0.0 if fam == "r2d2" else CLIP_ON
    eng, _, idx, npad = _learner(fam, clip)
    w0 = np.random.default_rng(10).standard_normal(idx.size).astype(np.float32) * 0.05
    st = _state(fam, idx.size, state)
    _load(fam, eng, w0, st)
    padded = _full(_crafted("random", idx.size, CLIP_ON), npad, idx)
    _write_bucket(eng, padded)
    if state == "rounding_step":
        assert int(f32(st["step"])) != st["step"] and st["step"] < FRAME
    end = SCHED["end_learning_rate"] if state == "end_rate" and fam != "r2d2" else None
    if end is not None:
        assert st["step"] >= FRAME
    _check(fam, eng, idx, npad, clip, padded, 1.0, state, expect_lr=end)


@pytest.mark.parametrize("fam", ADAM)
@pytest.mark.parametrize("gs", [1.0, 0.5, 0.125])
def test_grad_scale(native, fam, gs):
    clip = 0.0 if fam == "r2d2" else CLIP_ON
    eng, _, idx, npad = _learner(fam, clip)
    w0 = np.random.default_rng(11).standard_normal(idx.size).astype(np.float32) * 0.05
    _load(fam, eng, w0, _state(fam, idx.size, "restored"))
    padded = _full(_crafted("random", idx.size, CLIP_ON), npad, idx)
    _write_bucket(eng, padded)
    row = _check(fam, eng, idx, npad, clip, padded, gs, "gs=%g" % gs)
    if clip:
        assert row["grad_norm"] > clip


@pytest.mark.parametrize("fam", ["apex", "r2d2"])
def test_graph_apply_recaptures_on_grad_scale_change(native, fam):
    """Under use_cuda_graph the apply half is one captured graph per grad_scale: the sequence 1/2, 1/4, 1/2 captures it
    three times (learner_apply, graph_apply_scale) and must equal eager applies bit for bit."""
    clip = 0.0 if fam == "r2d2" else CLIP_ON
    engs = [_make(fam, clip, B=2, use_cuda_graph=g)[0] for g in (True, False)]
    try:
        idx, npad = op.bucket_index_map(engs[0])
        w0 = np.random.default_rng(12).standard_normal(idx.size).astype(np.float32) * 0.05
        st = _state(fam, idx.size, "restored")
        for e in engs:
            _load(fam, e, w0, st)
        for k, gs in enumerate((0.5, 0.25, 0.5)):
            padded = _full(_crafted("random", idx.size, CLIP_ON, seed=20 + k), npad, idx)
            rows, outs = [], []
            for e in engs:
                _write_bucket(e, padded)
                rows.append(_check(fam, e, idx, npad, clip, padded, gs, "graph gs=%g" % gs))
                outs.append(_read(fam, e))
            assert rows[0] == rows[1]
            for key in ("w", "m", "v"):
                assert np.array_equal(outs[0][key].view(np.uint32), outs[1][key].view(np.uint32)), (gs, key)
    finally:
        for e in engs:
            e.close()
