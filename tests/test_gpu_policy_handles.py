"""The IMPALA, R2D2, Ape-X and A3C policy engines share one core (csrc/policy_core.cuh).  What it promises, for every
engine: set_params / get_params refuse a wrong length and round-trip bitwise, last_act_ms needs a first act, the graph
and the eager engine compute the same bits over act, set_params, act, sync from a learner, act, and a sync from a
learner with another num_action is refused."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FAMILIES = ["impala", "r2d2", "apex", "a3c"]
PREFIX = {"impala": "policy", "r2d2": "r2d2_policy", "apex": "apex_policy", "a3c": "apex_policy"}   # drl_<prefix>_*
A = 4
N_ROWS = 5


@pytest.fixture(scope="module")
def gpu(native):
    if native.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return native


def _policy(family, graph):
    if family == "impala":
        from distributed_reinforcement_learning_b200.policy import NativePolicy
        return NativePolicy(8, num_action=A, use_cuda_graph=graph)
    if family == "r2d2":
        from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
        return NativeR2D2Policy(8, num_action=A, use_cuda_graph=graph)
    from distributed_reinforcement_learning_b200.apex_policy import NativeA3CPolicy, NativeApexPolicy
    return (NativeApexPolicy if family == "apex" else NativeA3CPolicy)(8, num_action=A, use_cuda_graph=graph)


def _learner(family, num_action=A):
    if family == "impala":
        from distributed_reinforcement_learning_b200.learner import NativeLearner
        return NativeLearner(batch=2, trajectory=4, num_action=num_action)
    if family == "r2d2":
        from distributed_reinforcement_learning_b200.r2d2_learner import NativeR2D2Learner
        return NativeR2D2Learner(batch=2, seq_len=6, burn_in=2, num_action=num_action)
    if family == "apex":
        from distributed_reinforcement_learning_b200.apex_learner import NativeApexLearner
        return NativeApexLearner(batch=4, num_action=num_action)
    from distributed_reinforcement_learning_b200.a3c_learner import NativeA3CLearner
    return NativeA3CLearner(batch=4, num_action=num_action)


def _params(p, seed):
    return (np.random.default_rng(seed).standard_normal(p.param_count) * 0.05).astype(np.float32)


def _act(p, family, seed):
    rng = np.random.default_rng(seed)
    st = rng.integers(0, 256, (N_ROWS,) + p.input_shape, dtype=np.uint8)
    pa = rng.integers(0, A, N_ROWS).astype(np.int32)
    if family in ("impala", "r2d2"):
        h = rng.standard_normal((N_ROWS, p.L)).astype(np.float32)
        c = rng.standard_normal((N_ROWS, p.L)).astype(np.float32)
        if family == "impala":
            return p.act(st, pa, h, c, uniform=rng.random(N_ROWS))
        return p.act(st, pa, h, c, explore_action=np.array([-1, 2, -1, 0, -1], np.int32))
    if family == "apex":
        return p.act(st, pa, explore_action=np.array([-1, 2, -1, 0, -1], np.int32))
    return p.act(st, pa, uniform=rng.random(N_ROWS))


@pytest.mark.parametrize("family", FAMILIES)
def test_params_wrong_length_and_round_trip(gpu, family):
    p = _policy(family, True)
    try:
        a = _params(p, 1)
        for fn in (getattr(gpu.lib, "drl_%s_set_params" % PREFIX[family]), getattr(gpu.lib, "drl_%s_get_params" % PREFIX[family])):
            for n in (a.size - 1, a.size + 1):
                assert fn(p._h, a.ctypes.data_as(C.c_void_p), n) == gpu.DRL_ERR_INVALID
        p.set_params(a)
        assert np.array_equal(p.get_params().view(np.uint32), a.view(np.uint32))
    finally:
        p.close()


@pytest.mark.parametrize("family", FAMILIES)
def test_last_act_ms_needs_an_act(gpu, family):
    p = _policy(family, True)
    try:
        ms = C.c_float()
        assert getattr(gpu.lib, "drl_%s_last_act_ms" % PREFIX[family])(p._h, C.byref(ms)) == gpu.DRL_ERR_STATE
        p.set_params(_params(p, 2))
        _act(p, family, 3)
        assert p.last_act_ms() > 0.0
    finally:
        p.close()


@pytest.mark.parametrize("family", FAMILIES)
def test_graph_and_eager_agree_bitwise_across_set_params_and_sync(gpu, family):
    pg, pe = _policy(family, True), _policy(family, False)
    learner = _learner(family)
    try:
        outs = {id(pg): [], id(pe): []}
        for p in (pg, pe):
            p.set_params(_params(p, 4))
            outs[id(p)].append(_act(p, family, 10))
            p.set_params(_params(p, 5))
            outs[id(p)].append(_act(p, family, 11))
        learner.set_params(_params(learner, 6))
        for p in (pg, pe):
            p.sync_from(learner)
            outs[id(p)].append(_act(p, family, 12))
            assert np.array_equal(p.get_params(), learner.get_params())
        for og, oe in zip(outs[id(pg)], outs[id(pe)]):
            assert og.keys() == oe.keys()
            for k in og:
                assert np.array_equal(np.asarray(og[k]).view(np.uint8), np.asarray(oe[k]).view(np.uint8)), k
    finally:
        for h in (pg, pe, learner):
            h.close()


@pytest.mark.parametrize("family", FAMILIES)
def test_sync_from_a_learner_with_another_num_action_is_refused(gpu, family):
    p = _policy(family, True)
    learner = _learner(family, num_action=A + 1)
    try:
        with pytest.raises(gpu.DrlError) as ei:
            p.sync_from(learner)
        assert ei.value.code == gpu.DRL_ERR_INVALID
    finally:
        p.close()
        learner.close()
