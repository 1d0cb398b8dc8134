"""CPU (no GPU needed): the device IMPALA trajectory queue and the policy recorder refuse to run without a device (no CPU
fallback), their argument checks that come before any device work, and VectorActor's refusal of a device queue that
does not fit its policy."""
import ctypes as C
import types

import numpy as np
import pytest


def _fake_queue(**kw):
    """A DeviceFIFOQueue's attributes without a device handle (the checks under test run before any device work)."""
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import DeviceFIFOQueue
    q = DeviceFIFOQueue.__new__(DeviceFIFOQueue)
    q.trajectory, q.input_shape, q.output_size, q.lstm_size = 20, (84, 84, 4), 18, 256
    q.batch_size, q.queue_size, q.device, q.max_rows = 32, 128, 0, 129
    q._q = C.c_void_p()
    for k, v in kw.items():
        setattr(q, k, v)
    return q


def _fake_policy(**kw):
    from distributed_reinforcement_learning_b200.policy import NativePolicy
    p = NativePolicy.__new__(NativePolicy)
    p.max_batch, p.A, p.L, p.input_shape, p.device = 64, 18, 256, (84, 84, 4), 0
    p._h = C.c_void_p()
    for k, v in kw.items():
        setattr(p, k, v)
    return p


class _Env:
    def reset(self):
        return np.zeros((84, 84, 4), np.uint8)


def test_queue_creation_fails_loudly_without_a_device(native):
    if native.device_count() > 0:
        pytest.skip("a CUDA device is present")
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import DeviceFIFOQueue
    with pytest.raises(native.DrlError) as ei:
        DeviceFIFOQueue(20, (84, 84, 4), 18, 128, 32, 20, 256)
    assert "no CPU fallback" in str(ei.value)
    assert ei.value.code == native.DRL_ERR_CUDA


def test_recorder_creation_fails_loudly_without_a_device(native):
    if native.device_count() > 0:
        pytest.skip("a CUDA device is present")
    N = native
    r = C.c_void_p()
    assert N.lib.drl_policy_recorder_create(None, None, 20, C.byref(r)) == N.DRL_ERR_CUDA
    assert "no CPU fallback" in N.lib.drl_last_error().decode()


def test_queue_rejects_bad_dimensions_before_looking_for_a_device(native):
    N = native
    q = C.c_void_p()
    for args in ((0, 84, 84, 4, 18, 256, 128, 32, 0), (20, 84, 84, 4, 18, 256, 16, 32, 0),
                 (20, 84, 84, 4, 0, 256, 128, 32, 0), (20, 84, 84, 4, 18, 256, 128, 0, 0)):
        assert N.lib.drl_traj_queue_create(*args, C.byref(q)) == N.DRL_ERR_INVALID
        assert "invalid dimensions" in N.lib.drl_last_error().decode()
    assert N.lib.drl_traj_queue_create(20, 84, 84, 4, 18, 256, 128, 32, 0, None) == N.DRL_ERR_INVALID
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import DeviceFIFOQueue
    with pytest.raises(ValueError, match="input_shape"):
        DeviceFIFOQueue(20, (84, 84), 18, 128, 32, 20, 256)


def test_entry_points_reject_null_handles(native):
    N = native
    z = np.zeros(64, np.float32)
    assert N.lib.drl_traj_queue_destroy(None) == N.DRL_OK
    assert N.lib.drl_traj_queue_size(None) == 0
    assert N.lib.drl_traj_queue_read(None, 0, *[N.ptr(z)] * 8) == N.DRL_ERR_INVALID
    assert "null trajectory queue handle" in N.lib.drl_last_error().decode()
    assert N.lib.drl_policy_recorder_destroy(None) == N.DRL_OK
    assert N.lib.drl_policy_recorder_act(None, *[N.ptr(z)] * 9) == N.DRL_ERR_INVALID
    assert "null recorder handle" in N.lib.drl_last_error().decode()
    assert N.lib.drl_policy_recorder_commit(None, N.ptr(z), N.ptr(z), -1) == N.DRL_ERR_INVALID
    assert N.lib.drl_policy_recorder_reset(None) == N.DRL_ERR_INVALID
    assert "null recorder handle" in N.lib.drl_last_error().decode()
    assert N.lib.drl_learner_stage_from_queue(None, 0, None, -1) == N.DRL_ERR_INVALID
    assert "null learner handle" in N.lib.drl_last_error().decode()


def test_recorder_python_side_validation(native):
    from distributed_reinforcement_learning_b200.policy import PolicyRecorder
    pol = _fake_policy()
    with pytest.raises(TypeError, match="DeviceFIFOQueue"):
        PolicyRecorder(pol, object(), 4)
    with pytest.raises(ValueError, match="n = 65"):
        PolicyRecorder(pol, _fake_queue(), 65)
    with pytest.raises(ValueError, match="n = 0"):
        PolicyRecorder(pol, _fake_queue(), 0)
    rec = PolicyRecorder.__new__(PolicyRecorder)
    rec.policy, rec.queue, rec.n, rec.T, rec._r = pol, _fake_queue(), 4, 20, C.c_void_p()
    st = np.zeros((4, 84, 84, 4), np.uint8)
    pa = np.zeros(4, np.int32)
    hc = np.zeros((4, 256), np.float32)
    with pytest.raises(ValueError, match="3 rows, the recorder records 4"):
        rec.act(st[:3], pa[:3], hc[:3], hc[:3])
    with pytest.raises(ValueError, match="state: expected uint8"):
        rec.act(st.astype(np.float32), pa, hc, hc)
    with pytest.raises(ValueError, match="previous_action: values"):
        rec.act(st, pa + 18, hc, hc)
    with pytest.raises(ValueError, match="h: expected shape"):
        rec.act(st, pa, hc[:, :64], hc)
    with pytest.raises(ValueError, match="uniform: draws"):
        rec.act(st, pa, hc, hc, uniform=np.ones(4))
    with pytest.raises(ValueError, match="reward: expected shape"):
        rec.commit(np.zeros((4, 19), np.float32), np.zeros((4, 20), np.bool_))
    with pytest.raises(ValueError, match="done: expected shape"):
        rec.commit(np.zeros((4, 20), np.float32), np.zeros((20, 4), np.bool_))


@pytest.mark.parametrize("kw,what", [(dict(trajectory=21), "steps"), (dict(output_size=6), "num_action"),
                                     (dict(lstm_size=64), "lstm"), (dict(input_shape=(84, 84, 1)), "frames"),
                                     (dict(device=1), "device"), (dict(max_rows=19), "at most 19")])
def test_vector_actor_rejects_a_device_queue_that_does_not_fit(native, kw, what):
    from distributed_reinforcement_learning_b200.actor import VectorActor
    with pytest.raises(ValueError, match=what):
        VectorActor(_fake_policy(), [_Env() for _ in range(20)], _fake_queue(**kw), 20, [18] * 20)


def test_vector_actor_rejects_more_environments_than_the_policy_serves(native):
    from distributed_reinforcement_learning_b200.actor import VectorActor
    with pytest.raises(ValueError, match="serves 1..16"):
        VectorActor(_fake_policy(max_batch=16), [_Env() for _ in range(20)], _fake_queue(), 20, [18] * 20)


def test_agent_and_queue_surface(native):
    from distributed_reinforcement_learning_b200.agent import impala
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import DeviceFIFOQueue
    from distributed_reinforcement_learning_b200.learner import NativeLearner
    from distributed_reinforcement_learning_b200.policy import NativePolicy
    assert callable(impala.Agent.train_from_queue)
    assert callable(NativeLearner.stage_from_queue)
    assert callable(NativePolicy.recorder)
    for name in ("get_size", "set_session", "close", "read"):
        assert callable(getattr(DeviceFIFOQueue, name))
    for name in ("append_to_queue", "sample_batch"):
        assert not hasattr(DeviceFIFOQueue, name)
    q = _fake_queue()
    q.set_session("s")
    assert q.sess == "s"
