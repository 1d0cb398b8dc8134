"""CPU (no GPU needed): the R2D2 device replay memory's C-ABI is exported and refuses to run without a device (no CPU
fallback), its argument checks that come before any device work, r2d2.Agent's device-memory surface, and
DeviceMemory.add's reduction of the stored (h, c) to step 0 and its chunking, against a stub replay."""
import threading

import numpy as np
import pytest


def test_replay_creation_fails_loudly_without_a_device(native):
    if native.device_count() > 0:
        pytest.skip("a CUDA device is present")
    from distributed_reinforcement_learning_b200.r2d2_replay import NativeR2D2Replay
    with pytest.raises(native.DrlError) as ei:
        NativeR2D2Replay(37, seq_len=6)
    assert "no CPU fallback" in str(ei.value)
    assert ei.value.code == native.DRL_ERR_CUDA


@pytest.mark.parametrize("kw,what", [(dict(capacity=1), "capacity"), (dict(capacity=0), "capacity"),
                                     (dict(capacity=-3), "capacity"), (dict(capacity=2 ** 31 + 1), "capacity"),
                                     (dict(seq_len=1), "seq_len"), (dict(seq_len=0), "seq_len"),
                                     (dict(input_shape=(84, 84, 3)), "channels"),
                                     (dict(num_action=1), "num_action"), (dict(num_action=33), "num_action")])
def test_replay_rejects_bad_arguments_before_looking_for_a_device(native, kw, what):
    from distributed_reinforcement_learning_b200.r2d2_replay import NativeR2D2Replay
    args = dict(capacity=37, seq_len=6, num_action=4, input_shape=(84, 84, 1))
    args.update(kw)
    with pytest.raises(native.DrlError) as ei:
        NativeR2D2Replay(**args)
    assert ei.value.code == native.DRL_ERR_INVALID and what in str(ei.value)


def test_replay_entry_points_reject_a_null_handle(native):
    import ctypes as C
    N = native
    u = np.zeros(64)
    for rc in (N.lib.drl_r2d2_replay_sample(None, 4, N.ptr(u), N.ptr(u), N.ptr(u), N.ptr(u), N.ptr(u)),
               N.lib.drl_r2d2_replay_update(None, 1, N.ptr(u), N.ptr(u)),
               N.lib.drl_r2d2_replay_last_sample(None, None, None, None),
               N.lib.drl_r2d2_replay_read(None, 0, 1, *[None] * 7),
               N.lib.drl_r2d2_replay_add(None, None, 1, *[N.ptr(u)] * 7, None),
               N.lib.drl_r2d2_replay_total(None, C.byref(C.c_double())),
               N.lib.drl_r2d2_replay_size(None, C.byref(C.c_int64())),
               N.lib.drl_r2d2_replay_beta(None, C.byref(C.c_double())),
               N.lib.drl_r2d2_replay_step_async(None, None, 0, N.ptr(u))):
        assert rc == N.DRL_ERR_INVALID
        assert "null r2d2 replay handle" in N.lib.drl_last_error().decode()
    assert N.lib.drl_r2d2_replay_destroy(None) == N.DRL_OK
    assert N.lib.drl_r2d2_replay_create(0, 37, 6, 1, 4, None) == N.DRL_ERR_INVALID


def test_agent_device_memory_surface(native):
    from distributed_reinforcement_learning_b200.agent import r2d2
    for name in ("device_memory", "train_from_memory"):
        assert callable(getattr(r2d2.Agent, name))
    for name in ("add", "total", "last_sample", "close"):
        assert callable(getattr(r2d2.DeviceMemory, name))
    assert r2d2.Agent.train_from_memory.__name__ == "train_from_memory"


class _StubReplay:
    def __init__(self):
        self.calls = []

    def add(self, learner, *fields):
        self.calls.append((learner, [np.array(f) for f in fields]))


class _StubAgent:
    def __init__(self, B):
        self._engine = type("Eng", (), {"B": B})()
        self._lock = threading.RLock()

    @staticmethod
    def _u8(state):
        from distributed_reinforcement_learning_b200.agent.r2d2 import Agent
        return Agent._u8(state)


def _memory(B):
    from distributed_reinforcement_learning_b200.agent import r2d2
    m = r2d2.DeviceMemory.__new__(r2d2.DeviceMemory)
    m.agent, m.capacity, m.replay = _StubAgent(B), 100, _StubReplay()
    return m


@pytest.mark.parametrize("stored_states", [True, False])
def test_device_memory_add_reduces_h_c_to_step_0_and_chunks(native, stored_states):
    rng = np.random.default_rng(0)
    n, S, L = 5, 3, 64
    state = rng.integers(0, 256, (n, S, 84, 84, 1), dtype=np.uint8)
    pa, ac = rng.integers(0, 4, (n, S)), rng.integers(0, 4, (n, S))
    h, c = rng.standard_normal((n, S, L)), rng.standard_normal((n, S, L))
    rw, dn = rng.standard_normal((n, S)).astype(np.float32), rng.random((n, S)) < 0.3
    m = _memory(2)
    if stored_states:
        m.add(state, pa, ac, h, c, rw, dn)
    else:
        m.add(list(state), pa, ac, h[:, 0], c[:, 0], rw, dn)
    calls = m.replay.calls
    assert [len(f[0]) for _, f in calls] == [2, 2, 1]            # chunks of the learner's batch, in order
    assert all(eng is m.agent._engine for eng, _ in calls)
    got = [np.concatenate([f[k] for _, f in calls]) for k in range(7)]
    assert np.array_equal(got[0], state)
    assert np.array_equal(got[1], pa) and np.array_equal(got[2], ac)
    assert got[3].dtype == np.float32 and got[3].shape == (n, L)
    assert np.array_equal(got[3], h[:, 0].astype(np.float32)) and np.array_equal(got[4], c[:, 0].astype(np.float32))
    assert np.array_equal(got[5], rw) and np.array_equal(got[6], dn)


def test_device_memory_add_refuses_float_frames(native):
    m = _memory(4)
    with pytest.raises(TypeError):
        m.add(np.zeros((1, 2, 84, 84, 1), np.float32), np.zeros((1, 2)), np.zeros((1, 2)), np.zeros((1, 64)),
              np.zeros((1, 64)), np.zeros((1, 2)), np.zeros((1, 2)))
