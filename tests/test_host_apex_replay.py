"""CPU (no GPU needed): the device replay memory's C-ABI is exported and refuses to run without a device (no CPU
fallback), its argument checks that come before any device work, and apex.Agent's device-memory surface."""
import numpy as np
import pytest


def test_replay_creation_fails_loudly_without_a_device(native):
    if native.device_count() > 0:
        pytest.skip("a CUDA device is present")
    from distributed_reinforcement_learning_b200.apex_replay import NativeApexReplay
    with pytest.raises(native.DrlError) as ei:
        NativeApexReplay(37)
    assert "no CPU fallback" in str(ei.value)
    assert ei.value.code == native.DRL_ERR_CUDA


def test_replay_rejects_a_capacity_below_two_before_looking_for_a_device(native):
    from distributed_reinforcement_learning_b200.apex_replay import NativeApexReplay
    for cap in (1, 0, -3):
        with pytest.raises(native.DrlError) as ei:
            NativeApexReplay(cap)
        assert ei.value.code == native.DRL_ERR_INVALID and "capacity" in str(ei.value)


def test_replay_entry_points_reject_a_null_handle(native):
    import ctypes as C
    N = native
    u = np.zeros(4)
    for rc in (N.lib.drl_apex_replay_sample(None, 4, N.ptr(u), N.ptr(u), N.ptr(u), N.ptr(u), N.ptr(u)),
               N.lib.drl_apex_replay_update(None, 1, N.ptr(u), N.ptr(u)),
               N.lib.drl_apex_replay_total(None, C.byref(C.c_double())),
               N.lib.drl_apex_replay_size(None, C.byref(C.c_int64())),
               N.lib.drl_apex_replay_step_async(None, None, 0, N.ptr(u))):
        assert rc == N.DRL_ERR_INVALID
    assert "null apex replay handle" in N.lib.drl_last_error().decode()
    assert N.lib.drl_apex_replay_destroy(None) == N.DRL_OK


def test_agent_device_memory_surface(native):
    from distributed_reinforcement_learning_b200.agent import apex
    for name in ("device_memory", "train_from_memory"):
        assert callable(getattr(apex.Agent, name))
    for name in ("add", "total", "last_sample", "close"):
        assert callable(getattr(apex.DeviceMemory, name))
