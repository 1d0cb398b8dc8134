"""CPU (no GPU needed): the entry points that the IMPALA, R2D2 and Ape-X / A3C policy engines share (csrc/policy_core.cuh)
reject a null handle with DRL_ERR_INVALID and the engine's own message, destroy(NULL) is a no-op, and param_count
refuses a null out-pointer."""
import ctypes as C

import pytest

FAMILIES = {"policy": "null policy handle", "r2d2_policy": "null r2d2 policy handle",
            "apex_policy": "null apex policy handle"}
ACT_ARGS = {"policy": 9, "r2d2_policy": 10, "apex_policy": 6}


def _calls(native, prefix):
    fn = lambda name: getattr(native.lib, "drl_%s_%s" % (prefix, name))   # noqa: E731
    ms = C.c_float()
    n = C.c_int64()
    buf = (C.c_float * 4)()
    calls = {
        "param_count": lambda: fn("param_count")(None, C.byref(n)),
        "set_params": lambda: fn("set_params")(None, buf, 4),
        "get_params": lambda: fn("get_params")(None, buf, 4),
        "sync_from_learner": lambda: fn("sync_from_learner")(None, None),
        "last_act_ms": lambda: fn("last_act_ms")(None, C.byref(ms)),
        "act": lambda: fn("act")(None, 1, *([None] * ACT_ARGS[prefix])),
    }
    if prefix == "apex_policy":
        calls["a3c_act"] = lambda: native.lib.drl_a3c_policy_act(None, 1, *([None] * 6))
    return calls


@pytest.mark.parametrize("prefix", sorted(FAMILIES))
def test_null_handle_is_rejected_with_the_family_message(native, prefix):
    for name, call in _calls(native, prefix).items():
        assert call() == native.DRL_ERR_INVALID, (prefix, name)
        assert native.lib.drl_last_error().decode() == FAMILIES[prefix], (prefix, name)


@pytest.mark.parametrize("prefix", sorted(FAMILIES))
def test_destroy_null_is_a_no_op(native, prefix):
    assert getattr(native.lib, "drl_%s_destroy" % prefix)(None) == native.DRL_OK


@pytest.mark.parametrize("prefix", sorted(FAMILIES))
def test_param_count_rejects_a_null_out_pointer(native, prefix):
    assert getattr(native.lib, "drl_%s_param_count" % prefix)(None, None) == native.DRL_ERR_INVALID
