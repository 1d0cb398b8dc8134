"""CPU (no GPU needed): the device R2D2 sequence queue and the R2D2 policy recorder refuse to run without a device (no
CPU fallback), their argument checks that come before any device work, R2D2VectorActor's refusal of a device queue
that does not fit its policy, DeviceMemory.add_from_queue's checks, and the surface of the new Python API."""
import ctypes as C
import threading

import numpy as np
import pytest


def _fake_queue(**kw):
    """An R2D2DeviceFIFOQueue's attributes without a device handle (the checks under test run before any device
    work)."""
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import R2D2DeviceFIFOQueue
    q = R2D2DeviceFIFOQueue.__new__(R2D2DeviceFIFOQueue)
    q.seq_len, q.input_shape, q.output_size, q.lstm_size = 15, (84, 84, 1), 4, 64
    q.batch_size, q.queue_size, q.device, q.max_rows = 16, 128, 0, 129
    q._q = C.c_void_p()
    for k, v in kw.items():
        setattr(q, k, v)
    return q


def _fake_policy(**kw):
    from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
    p = NativeR2D2Policy.__new__(NativeR2D2Policy)
    p.max_batch, p.A, p.L, p.input_shape, p.device = 64, 4, 64, (84, 84, 1), 0
    p._h = C.c_void_p()
    for k, v in kw.items():
        setattr(p, k, v)
    return p


class _Env:
    def reset(self):
        return np.zeros((84, 84, 1), np.uint8)


def test_queue_creation_fails_loudly_without_a_device(native):
    if native.device_count() > 0:
        pytest.skip("a CUDA device is present")
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import R2D2DeviceFIFOQueue
    with pytest.raises(native.DrlError) as ei:
        R2D2DeviceFIFOQueue(15, (84, 84, 1), 4, 128, 16, 40, 64)
    assert "no CPU fallback" in str(ei.value)
    assert ei.value.code == native.DRL_ERR_CUDA


def test_recorder_creation_fails_loudly_without_a_device(native):
    if native.device_count() > 0:
        pytest.skip("a CUDA device is present")
    N = native
    r = C.c_void_p()
    assert N.lib.drl_r2d2_policy_recorder_create(None, None, 16, C.byref(r)) == N.DRL_ERR_CUDA
    assert "no CPU fallback" in N.lib.drl_last_error().decode()


def test_queue_rejects_bad_dimensions_before_looking_for_a_device(native):
    N = native
    q = C.c_void_p()
    for args, what in (((1, 1, 4, 128, 16, 0), "seq_len"), ((15, 3, 4, 128, 16, 0), "channels"),
                       ((15, 1, 1, 128, 16, 0), "num_action"), ((15, 1, 33, 128, 16, 0), "num_action"),
                       ((15, 1, 4, 8, 16, 0), "invalid dimensions"), ((15, 1, 4, 128, 0, 0), "invalid dimensions"),
                       ((15, 1, 4, 128, 16, 99), "no CPU fallback")):
        rc = N.lib.drl_r2d2_queue_create(*args, C.byref(q))
        assert rc == (N.DRL_ERR_CUDA if what == "no CPU fallback" else N.DRL_ERR_INVALID), args
        assert what in N.lib.drl_last_error().decode()
    assert N.lib.drl_r2d2_queue_create(15, 1, 4, 128, 16, 0, None) == N.DRL_ERR_INVALID
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import R2D2DeviceFIFOQueue
    with pytest.raises(ValueError, match="input_shape"):
        R2D2DeviceFIFOQueue(15, (84, 84), 4, 128, 16, 40, 64)
    with pytest.raises(ValueError, match="input_shape"):
        R2D2DeviceFIFOQueue(15, (64, 64, 1), 4, 128, 16, 40, 64)
    with pytest.raises(ValueError, match="lstm_size"):
        R2D2DeviceFIFOQueue(15, (84, 84, 1), 4, 128, 16, 40, 256)


def test_entry_points_reject_null_handles(native):
    N = native
    z = np.zeros(64, np.float32)
    assert N.lib.drl_r2d2_queue_destroy(None) == N.DRL_OK
    assert N.lib.drl_r2d2_queue_size(None) == 0
    assert N.lib.drl_r2d2_queue_read(None, 0, *[N.ptr(z)] * 7) == N.DRL_ERR_INVALID
    assert "null r2d2 queue handle" in N.lib.drl_last_error().decode()
    assert N.lib.drl_r2d2_policy_recorder_destroy(None) == N.DRL_OK
    assert N.lib.drl_r2d2_policy_recorder_act(None, *[N.ptr(z)] * 10) == N.DRL_ERR_INVALID
    assert "null recorder handle" in N.lib.drl_last_error().decode()
    assert N.lib.drl_r2d2_policy_recorder_commit(None, N.ptr(z), N.ptr(z), -1) == N.DRL_ERR_INVALID
    assert "null recorder handle" in N.lib.drl_last_error().decode()
    assert N.lib.drl_r2d2_policy_recorder_reset(None) == N.DRL_ERR_INVALID
    assert "null recorder handle" in N.lib.drl_last_error().decode()
    assert N.lib.drl_r2d2_replay_add_from_queue(None, None, None, -1) == N.DRL_ERR_INVALID
    assert "null r2d2 replay handle" in N.lib.drl_last_error().decode()


def test_recorder_python_side_validation(native):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import DeviceFIFOQueue
    from distributed_reinforcement_learning_b200.r2d2_policy import R2D2PolicyRecorder
    pol = _fake_policy()
    with pytest.raises(TypeError, match="R2D2DeviceFIFOQueue"):
        R2D2PolicyRecorder(pol, object(), 4)
    with pytest.raises(TypeError, match="R2D2DeviceFIFOQueue"):
        R2D2PolicyRecorder(pol, DeviceFIFOQueue.__new__(DeviceFIFOQueue), 4)
    with pytest.raises(ValueError, match="n = 65"):
        R2D2PolicyRecorder(pol, _fake_queue(), 65)
    with pytest.raises(ValueError, match="n = 0"):
        R2D2PolicyRecorder(pol, _fake_queue(), 0)
    rec = R2D2PolicyRecorder.__new__(R2D2PolicyRecorder)
    rec.policy, rec.queue, rec.n, rec.T, rec._r = pol, _fake_queue(), 4, 15, C.c_void_p()
    st = np.zeros((4, 84, 84, 1), np.uint8)
    pa = np.zeros(4, np.int32)
    hc = np.zeros((4, 64), np.float32)
    with pytest.raises(ValueError, match="3 rows, the recorder records 4"):
        rec.act(st[:3], pa[:3], hc[:3], hc[:3])
    with pytest.raises(ValueError, match="state: expected uint8"):
        rec.act(st.astype(np.float32), pa, hc, hc)
    with pytest.raises(ValueError, match="previous_action: values"):
        rec.act(st, pa + 4, hc, hc)
    with pytest.raises(ValueError, match="h: expected shape"):
        rec.act(st, pa, np.zeros((4, 256), np.float32), hc)
    with pytest.raises(ValueError, match="explore_action: values"):
        rec.act(st, pa, hc, hc, explore_action=np.full(4, 4))
    with pytest.raises(ValueError, match="epsilon or explore_action"):
        rec.act(st, pa, hc, hc, epsilon=0.5, explore_action=np.zeros(4, np.int32))
    with pytest.raises(ValueError, match="reward: expected shape"):
        rec.commit(np.zeros((4, 14), np.float32), np.zeros((4, 15), np.bool_))
    with pytest.raises(ValueError, match="done: expected shape"):
        rec.commit(np.zeros((4, 15), np.float32), np.zeros((15, 4), np.bool_))


@pytest.mark.parametrize("kw,what", [(dict(seq_len=16), "steps"), (dict(output_size=6), "num_action"),
                                     (dict(lstm_size=256), "lstm"), (dict(input_shape=(84, 84, 4)), "frames"),
                                     (dict(device=1), "device"), (dict(max_rows=19), "at most 19")])
def test_vector_actor_rejects_a_device_queue_that_does_not_fit(native, kw, what):
    from distributed_reinforcement_learning_b200.actor import R2D2VectorActor
    with pytest.raises(ValueError, match=what):
        R2D2VectorActor(_fake_policy(), [_Env() for _ in range(20)], _fake_queue(**kw), 15)


def test_vector_actor_rejects_more_environments_than_the_policy_serves(native):
    from distributed_reinforcement_learning_b200.actor import R2D2VectorActor
    with pytest.raises(ValueError, match="serves 1..16"):
        R2D2VectorActor(_fake_policy(max_batch=16), [_Env() for _ in range(20)], _fake_queue(), 15)


def _agent():
    from distributed_reinforcement_learning_b200.agent import r2d2
    return r2d2.Agent(seq_len=15, burn_in=7, input_shape=(84, 84, 1), num_action=4, lstm_size=64,
                      discount_factor=0.997, start_learning_rate=1e-4, end_learning_rate=0.0, learning_frame=1e9,
                      gradient_clip_norm=40.0, model_name="host_q", learner_name="host_q")


def test_add_from_queue_python_side_validation(native, monkeypatch):
    from distributed_reinforcement_learning_b200 import dp
    from distributed_reinforcement_learning_b200.agent import r2d2
    from distributed_reinforcement_learning_b200.r2d2_replay import NativeR2D2Replay
    rep = NativeR2D2Replay.__new__(NativeR2D2Replay)
    rep._h = C.c_void_p()
    with pytest.raises(TypeError, match="R2D2DeviceFIFOQueue"):
        rep.add_from_queue(None, object())
    mem = r2d2.DeviceMemory.__new__(r2d2.DeviceMemory)
    mem.agent, mem.replay = _agent(), rep
    monkeypatch.setattr(dp, "distributed", lambda: True)
    with pytest.raises(RuntimeError, match="local to one GPU"):
        mem.add_from_queue(_fake_queue())


def test_add_from_queue_waits_without_the_agents_lock(native):
    """The pop blocks inside the C call; actor threads take the agent's lock in sync_policy meanwhile."""
    from distributed_reinforcement_learning_b200.agent import r2d2
    ag = _agent()
    ag._engine = object()
    held = []

    class SpyReplay:
        def add_from_queue(self, eng, queue, timeout_ms):
            def other_thread():
                got = ag._lock.acquire(timeout=1.0)
                held.append(got)
                if got:
                    ag._lock.release()
            t = threading.Thread(target=other_thread)
            t.start()
            t.join()
            held.append((eng, queue, timeout_ms))

    mem = r2d2.DeviceMemory.__new__(r2d2.DeviceMemory)
    mem.agent, mem.replay = ag, SpyReplay()
    q = _fake_queue()
    mem.add_from_queue(q, timeout_ms=7)
    assert held[0] is True and held[1] == (ag._engine, q, 7)


def test_surface(native):
    from distributed_reinforcement_learning_b200.agent import r2d2
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import R2D2DeviceFIFOQueue
    from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
    from distributed_reinforcement_learning_b200.r2d2_replay import NativeR2D2Replay
    assert callable(r2d2.DeviceMemory.add_from_queue)
    assert callable(NativeR2D2Replay.add_from_queue)
    assert callable(NativeR2D2Policy.recorder)
    for name in ("get_size", "set_session", "close", "read"):
        assert callable(getattr(R2D2DeviceFIFOQueue, name))
    for name in ("append_to_queue", "sample_batch"):
        assert not hasattr(R2D2DeviceFIFOQueue, name)
    q = _fake_queue()
    q.set_session("s")
    assert q.sess == "s"
    assert q.max_rows == 129 and q.batch_size == 16
    for name in ("drl_r2d2_queue_create", "drl_r2d2_queue_destroy", "drl_r2d2_queue_size", "drl_r2d2_queue_read",
                 "drl_r2d2_policy_recorder_create", "drl_r2d2_policy_recorder_destroy", "drl_r2d2_policy_recorder_act",
                 "drl_r2d2_policy_recorder_commit", "drl_r2d2_policy_recorder_reset",
                 "drl_r2d2_replay_add_from_queue"):
        assert name in native.EXPORTS
