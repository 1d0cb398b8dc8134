"""The IMPALA, Ape-X, A3C and R2D2 handles share one core (csrc/learner_core.cuh).  What it promises, for every family at
small shapes: the CUDA-graph and the eager step compute the same bits, the data-parallel halves (forward_backward +
apply, graph or eager) compute what one step computes, parameter and optimizer state round-trip bitwise, and each
misuse of the C-ABI fails with the same error code."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FAMILIES = ["learner", "apex", "a3c", "r2d2"]
A = 4


def _learner(family, use_cuda_graph):
    if family == "learner":
        from distributed_reinforcement_learning_b200.learner import NativeLearner
        return NativeLearner(batch=2, trajectory=5, num_action=A, use_cuda_graph=use_cuda_graph)
    if family == "apex":
        from distributed_reinforcement_learning_b200.apex_learner import NativeApexLearner
        return NativeApexLearner(batch=4, num_action=A, use_cuda_graph=use_cuda_graph)
    if family == "a3c":
        from distributed_reinforcement_learning_b200.a3c_learner import NativeA3CLearner
        return NativeA3CLearner(batch=4, num_action=A, use_cuda_graph=use_cuda_graph)
    from distributed_reinforcement_learning_b200.r2d2_learner import NativeR2D2Learner
    return NativeR2D2Learner(batch=2, seq_len=6, burn_in=2, num_action=A, use_cuda_graph=use_cuda_graph)


def _init(eng, seed=0):
    rng = np.random.default_rng(seed)
    if eng.family in ("learner", "a3c"):
        eng.set_params(rng.standard_normal(eng.param_count).astype(np.float32) * 0.05)
        return
    for which in (0, 1):
        eng.set_params(rng.standard_normal(eng.param_count).astype(np.float32) * 0.05, which)


def _batch(eng, seed):
    rng = np.random.default_rng(seed)
    B = eng.B
    if eng.family == "learner":
        T = eng.T
        mu = rng.random((B, T, A)).astype(np.float32) + 0.1
        return (rng.integers(0, 256, (B, T) + eng.input_shape, dtype=np.uint8), rng.standard_normal((B, T)),
                rng.integers(0, A, (B, T)), rng.random((B, T)) < 0.2, mu / mu.sum(-1, keepdims=True),
                rng.integers(0, A, (B, T)), rng.standard_normal((B, T, eng.L)).astype(np.float32) * 0.1,
                rng.standard_normal((B, T, eng.L)).astype(np.float32) * 0.1)
    if eng.family == "r2d2":
        S = eng.S
        return (rng.integers(0, 256, (B, S) + eng.input_shape, dtype=np.uint8), rng.integers(0, A, (B, S)),
                rng.integers(0, A, (B, S)), rng.standard_normal((B, eng.L)).astype(np.float32) * 0.1,
                rng.standard_normal((B, eng.L)).astype(np.float32) * 0.1, rng.standard_normal((B, S)),
                rng.random((B, S)) < 0.2, rng.uniform(0.5, 1.5, B))
    frames = [rng.integers(0, 256, (B,) + eng.input_shape, dtype=np.uint8) for _ in range(2)]
    rest = (rng.integers(0, A, B), rng.integers(0, A, B), rng.standard_normal(B) * 2, rng.random(B) < 0.2)
    return tuple(frames) + rest + (() if eng.family == "a3c" else (rng.uniform(0.5, 1.5, B),))


def _sync_target(eng):
    if eng.family == "apex":
        eng.target_to_main()          # target <- main (sic)
    elif eng.family == "r2d2":
        eng.main_to_target()


def _scalars(out):
    out, td = out if isinstance(out, tuple) else (out, None)
    return {k: np.float32(v) if isinstance(v, float) else v for k, v in out.items()}, td


def _state(eng):
    opt = eng.get_opt_state()
    if eng.family == "learner":
        opt = dict(ms=opt[0], step=opt[1])
    s = dict(grads=eng.get_grads(), **{"opt_" + k: v for k, v in opt.items()})
    s["taps"] = eng.taps()
    if eng.family in ("learner", "a3c"):
        s["params"] = eng.get_params()
    else:
        s["params"], s["target"] = eng.get_params(0), eng.get_params(1)
    return s


def _assert_same(a, b, where=""):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), where
        for k in a:
            _assert_same(a[k], b[k], "%s.%s" % (where, k))
    elif isinstance(a, tuple):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _assert_same(x, y, "%s[%d]" % (where, i))
    elif a is None:
        assert b is None, where
    else:
        x, y = np.asarray(a), np.asarray(b)
        assert x.shape == y.shape and x.dtype == y.dtype, where
        assert x.tobytes() == y.tobytes(), where


def _run(eng, steps, sync_after=None):
    outs = []
    for i in range(steps):
        eng.stage(i % 2, *_batch(eng, 10 + i))
        outs.append(_scalars(eng.step(i % 2)))
        if i == sync_after:
            _sync_target(eng)
    return outs


@pytest.mark.parametrize("family", FAMILIES)
def test_graph_and_eager_steps_match_bitwise(native, family):
    res = []
    for graph in (True, False):
        eng = _learner(family, graph)
        try:
            _init(eng)
            outs = _run(eng, 3, sync_after=1)
            res.append((outs, _state(eng)))
        finally:
            eng.close()
    (o1, s1), (o2, s2) = res
    for i, (a, b) in enumerate(zip(o1, o2)):
        _assert_same(a[0], b[0], "step%d.scalars" % i)
        _assert_same(a[1], b[1], "step%d.td_error" % i)
    _assert_same(s1, s2)


def _apply(native, eng):
    if eng.family == "learner":       # no grad_scale: the IMPALA losses are batch sums
        native.check(eng._fn("apply")(eng._h))
    else:
        native.check(eng._fn("apply")(eng._h, C.c_float(1.0)))


@pytest.mark.parametrize("use_cuda_graph", [False, True])
@pytest.mark.parametrize("family", FAMILIES)
def test_forward_backward_then_apply_matches_step(native, family, use_cuda_graph):
    ref = _learner(family, use_cuda_graph)
    eng = _learner(family, use_cuda_graph)
    try:
        for e in (ref, eng):
            _init(e)
        for i in range(3):            # a graph replays from the second call on
            for e in (ref, eng):
                e.stage(i % 2, *_batch(e, 3 + i))
            want = _scalars(ref.step(i % 2))
            native.check(eng._fn("forward_backward")(eng._h, i % 2))
            _apply(native, eng)
            got = _scalars(eng.wait())
            _assert_same(want, got, "step%d" % i)
            _assert_same(_state(ref), _state(eng), "step%d" % i)
    finally:
        ref.close()
        eng.close()


@pytest.mark.parametrize("family", FAMILIES)
def test_params_and_opt_state_round_trip(native, family):
    eng = _learner(family, False)
    rng = np.random.default_rng(1)
    try:
        whiches = [()] if family in ("learner", "a3c") else [(0,), (1,)]
        for which in whiches:
            p = rng.standard_normal(eng.param_count).astype(np.float32)
            eng.set_params(p, *which)
            assert eng.get_params(*which).tobytes() == p.tobytes()
        if family == "learner":       # RMSProp: the ms slots and global_step
            ms = rng.random(eng.param_count).astype(np.float32)
            eng.set_opt_state(ms, 12345678901)
            got, step = eng.get_opt_state()
            assert got.tobytes() == ms.tobytes() and step == 12345678901
            return
        m = rng.standard_normal(eng.param_count).astype(np.float32)
        v = rng.random(eng.param_count).astype(np.float32)
        eng.set_opt_state(m, v, 12345678901, 0.25, 0.5)
        st = eng.get_opt_state()
        assert st["m"].tobytes() == m.tobytes() and st["v"].tobytes() == v.tobytes()
        assert (st["step"], st["beta1_power"], st["beta2_power"]) == (12345678901, 0.25, 0.5)
    finally:
        eng.close()


@pytest.mark.parametrize("family", FAMILIES)
def test_misuse_fails_with_the_same_code(native, family):
    fn = lambda name: getattr(native.lib, "drl_%s_%s" % (family, name))   # noqa: E731

    def code(rc):
        assert rc != native.DRL_OK
        return rc

    assert code(fn("step_async")(None, 0)) == native.DRL_ERR_INVALID
    name = family if family in ("learner", "r2d2") else "apex"
    assert "null %s handle" % name in native.lib.drl_last_error().decode()
    eng = _learner(family, False)
    try:
        h, n = eng._h, eng.param_count
        buf = np.zeros(n + 1, np.float32)
        assert code(fn("step_async")(h, eng.num_slots)) == native.DRL_ERR_INVALID          # slot out of range
        assert code(fn("forward_backward")(h, -1)) == native.DRL_ERR_INVALID
        assert code(fn("step_async")(h, 0)) == native.DRL_ERR_STATE                       # slot not staged
        assert code(fn("forward_backward")(h, 0)) == native.DRL_ERR_STATE
        with pytest.raises(native.DrlError) as ei:
            eng.wait()                                                                    # nothing in flight
        assert ei.value.code == native.DRL_ERR_STATE
        assert code(fn("get_grads")(h, native.ptr(buf), n + 1)) == native.DRL_ERR_INVALID  # wrong length
        if family == "learner":
            assert code(fn("get_opt_state")(h, None, n - 1, None)) == native.DRL_ERR_INVALID
            assert code(fn("wait_slot")(h, eng.num_slots, None)) == native.DRL_ERR_INVALID
        else:
            assert code(fn("get_opt_state")(h, None, None, n - 1, None, None, None)) == native.DRL_ERR_INVALID
        if family in ("learner", "a3c"):
            assert code(fn("set_params")(h, native.ptr(buf), n + 1)) == native.DRL_ERR_INVALID
        else:
            assert code(fn("set_params")(h, 0, native.ptr(buf), n + 1)) == native.DRL_ERR_INVALID
            assert code(fn("get_params")(h, 2, native.ptr(buf), n)) == native.DRL_ERR_INVALID   # bad which
        if family != "learner":
            assert code(fn("apply")(h, C.c_float(0.0))) == native.DRL_ERR_INVALID          # grad_scale <= 0
            assert code(fn("apply")(h, C.c_float(-1.0))) == native.DRL_ERR_INVALID
        if family == "apex":
            assert code(native.lib.drl_a3c_step_async(h, 0)) == native.DRL_ERR_INVALID
            assert "not an A3C handle" in native.lib.drl_last_error().decode()
    finally:
        eng.close()
