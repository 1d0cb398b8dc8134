"""CPU (no GPU needed): the device Ape-X transition queue and the device actor buffers refuse to run without a device
(no CPU fallback), their argument checks that come before any device work, ApexVectorActor's refusal of a device queue
that does not fit its policy, DeviceMemory.add_from_queue's checks and its wait without the agent's lock, and the
surface of the new Python API."""
import ctypes as C
import threading

import numpy as np
import pytest

T, A = 32, 6
SHAPE = (84, 84, 4)


def _fake_queue(**kw):
    """An ApexDeviceFIFOQueue's attributes without a device handle (the checks under test run before any device
    work)."""
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import ApexDeviceFIFOQueue
    q = ApexDeviceFIFOQueue.__new__(ApexDeviceFIFOQueue)
    q.trajectory, q.input_shape, q.output_size = T, SHAPE, A
    q.batch_size, q.queue_size, q.num_actors, q.device = 32, 32, 20, 0
    q._q = C.c_void_p()
    for k, v in kw.items():
        setattr(q, k, v)
    return q


def _fake_policy(**kw):
    from distributed_reinforcement_learning_b200.apex_policy import NativeApexPolicy
    p = NativeApexPolicy.__new__(NativeApexPolicy)
    p.max_batch, p.A, p.input_shape, p.device = 64, A, SHAPE, 0
    p._h = C.c_void_p()
    for k, v in kw.items():
        setattr(p, k, v)
    return p


class _Env:
    def reset(self):
        return np.zeros(SHAPE, np.uint8)


def test_creation_fails_loudly_without_a_device(native):
    if native.device_count() > 0:
        pytest.skip("a CUDA device is present")
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import (ApexDeviceFIFOQueue,
                                                                                         DeviceLocalBuffers)
    with pytest.raises(native.DrlError) as ei:
        ApexDeviceFIFOQueue(T, SHAPE, A, 32, 32, 20)
    assert "no CPU fallback" in str(ei.value) and ei.value.code == native.DRL_ERR_CUDA
    with pytest.raises(native.DrlError) as ei:
        DeviceLocalBuffers(20, 10000, A)
    assert "no CPU fallback" in str(ei.value) and ei.value.code == native.DRL_ERR_CUDA


def test_arguments_are_checked_before_looking_for_a_device(native):
    N = native
    q = C.c_void_p()
    for args, what in (((0, A, 32, 0), "trajectory"), ((513, A, 32, 0), "trajectory"), ((T, 1, 32, 0), "num_action"),
                       ((T, 33, 32, 0), "num_action"), ((T, A, 0, 0), "capacity"), ((T, A, 32, 99), "no CPU fallback")):
        rc = N.lib.drl_apex_queue_create(*args, C.byref(q))
        assert rc == (N.DRL_ERR_CUDA if what == "no CPU fallback" else N.DRL_ERR_INVALID), args
        assert what in N.lib.drl_last_error().decode()
    assert N.lib.drl_apex_queue_create(T, A, 32, 0, None) == N.DRL_ERR_INVALID
    b = C.c_void_p()
    for args, what in (((0, 100, A, 0), "n must"), ((4, 1, A, 0), "capacity"), ((4, 100, 1, 0), "num_action"),
                       ((4, 100, 33, 0), "num_action"), ((4, 100, A, 99), "no CPU fallback")):
        rc = N.lib.drl_apex_actor_buffer_create(*args, C.byref(b))
        assert rc == (N.DRL_ERR_CUDA if what == "no CPU fallback" else N.DRL_ERR_INVALID), args
        assert what in N.lib.drl_last_error().decode()
    assert N.lib.drl_apex_actor_buffer_create(4, 100, A, 0, None) == N.DRL_ERR_INVALID
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import ApexDeviceFIFOQueue
    with pytest.raises(ValueError, match="input_shape"):
        ApexDeviceFIFOQueue(T, (84, 84, 1), A, 32, 32, 20)


def test_entry_points_reject_null_handles(native):
    N = native
    z = np.zeros(SHAPE, np.uint8)
    assert N.lib.drl_apex_queue_destroy(None) == N.DRL_OK
    assert N.lib.drl_apex_queue_size(None) == 0
    assert N.lib.drl_apex_queue_read(None, 0, *[N.ptr(z)] * 6) == N.DRL_ERR_INVALID
    assert "null apex queue handle" in N.lib.drl_last_error().decode()
    assert N.lib.drl_apex_actor_buffer_destroy(None) == N.DRL_OK
    n = C.c_int64()
    assert N.lib.drl_apex_actor_buffer_size(None, C.byref(n)) == N.DRL_ERR_INVALID
    assert "null apex actor buffer handle" in N.lib.drl_last_error().decode()
    assert N.lib.drl_apex_actor_buffer_append(None, 1, *[N.ptr(z)] * 6) == N.DRL_ERR_INVALID
    assert "null apex actor buffer handle" in N.lib.drl_last_error().decode()
    assert N.lib.drl_apex_actor_buffer_push(None, None, 0, N.ptr(z), -1) == N.DRL_ERR_INVALID
    assert "null apex actor buffer handle" in N.lib.drl_last_error().decode()
    assert N.lib.drl_apex_actor_buffer_read(None, 0, 0, *[N.ptr(z)] * 6) == N.DRL_ERR_INVALID
    assert "null apex actor buffer handle" in N.lib.drl_last_error().decode()
    assert N.lib.drl_apex_replay_add_from_queue(None, None, None, -1) == N.DRL_ERR_INVALID
    assert "null apex replay handle" in N.lib.drl_last_error().decode()


def test_device_buffers_python_side_validation(native):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import (DeviceFIFOQueue,
                                                                                         DeviceLocalBuffers)
    b = DeviceLocalBuffers.__new__(DeviceLocalBuffers)
    b.n, b.capacity, b.num_action, b.device, b._b = 4, 200, A, 0, C.c_void_p()
    st = np.zeros((4,) + SHAPE, np.uint8)
    z = np.zeros(4)
    with pytest.raises(ValueError, match="state: expected shape"):
        b.append(st[:3], st, z, z, z, z)
    with pytest.raises(ValueError, match="next_state: expected shape"):
        b.append(st, st[:, :80], z, z, z, z)
    with pytest.raises(ValueError, match="reward: expected shape"):
        b.append(st, st, z, z, np.zeros(5), z)
    with pytest.raises(ValueError, match="previous_action: values"):
        b.append(st, st, z + A, z, z, z)
    with pytest.raises(ValueError, match="action: values"):
        b.append(st, st, z, z - 1, z, z)
    with pytest.raises(TypeError, match="ApexDeviceFIFOQueue"):
        b.push(object(), 0, np.arange(T))
    with pytest.raises(TypeError, match="ApexDeviceFIFOQueue"):
        b.push(DeviceFIFOQueue.__new__(DeviceFIFOQueue), 0, np.arange(T))
    with pytest.raises(ValueError, match="order: expected shape"):
        b.push(_fake_queue(), 0, np.arange(T - 1))
    for bad in (np.arange(T) - 1, np.arange(T) + 200 - T + 1):
        with pytest.raises(ValueError, match="order: deque indices"):
            b.push(_fake_queue(), 0, bad)


@pytest.mark.parametrize("kw,what", [(dict(trajectory=16), "transitions"), (dict(output_size=4), "num_action"),
                                     (dict(device=1), "device")])
def test_vector_actor_rejects_a_device_queue_that_does_not_fit(native, kw, what):
    from distributed_reinforcement_learning_b200.actor import ApexVectorActor
    with pytest.raises(ValueError, match=what):
        ApexVectorActor(_fake_policy(), [_Env() for _ in range(20)], _fake_queue(**kw), T, [A] * 20)


def _agent():
    from distributed_reinforcement_learning_b200.agent import apex
    return apex.Agent(input_shape=SHAPE, num_action=A, discount_factor=0.99, gradient_clip_norm=40.0,
                      reward_clipping="abs_one", start_learning_rate=1e-4, end_learning_rate=0.0,
                      learning_frame=1e9, model_name="host_aq", learner_name="host_aq")


def test_add_from_queue_python_side_validation(native, monkeypatch):
    from distributed_reinforcement_learning_b200 import dp
    from distributed_reinforcement_learning_b200.agent import apex
    from distributed_reinforcement_learning_b200.apex_replay import NativeApexReplay
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import R2D2DeviceFIFOQueue
    rep = NativeApexReplay.__new__(NativeApexReplay)
    rep._h = C.c_void_p()
    with pytest.raises(TypeError, match="ApexDeviceFIFOQueue"):
        rep.add_from_queue(None, object())
    with pytest.raises(TypeError, match="ApexDeviceFIFOQueue"):
        rep.add_from_queue(None, R2D2DeviceFIFOQueue.__new__(R2D2DeviceFIFOQueue))
    mem = apex.DeviceMemory.__new__(apex.DeviceMemory)
    mem.agent, mem.replay = _agent(), rep
    monkeypatch.setattr(dp, "distributed", lambda: True)
    with pytest.raises(RuntimeError, match="local to one GPU"):
        mem.add_from_queue(_fake_queue())


def test_add_from_queue_waits_without_the_agents_lock(native):
    """The pop blocks inside the C call; actor threads take the agent's lock in sync_policy meanwhile."""
    from distributed_reinforcement_learning_b200.agent import apex
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

    mem = apex.DeviceMemory.__new__(apex.DeviceMemory)
    mem.agent, mem.replay = ag, SpyReplay()
    q = _fake_queue()
    mem.add_from_queue(q, timeout_ms=7)
    assert held[0] is True and held[1] == (ag._engine, q, 7)


def test_surface(native):
    from distributed_reinforcement_learning_b200.agent import apex
    from distributed_reinforcement_learning_b200.apex_replay import NativeApexReplay
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import (ApexDeviceFIFOQueue,
                                                                                         DeviceLocalBuffers)
    assert callable(apex.DeviceMemory.add_from_queue)
    assert callable(NativeApexReplay.add_from_queue)
    for name in ("get_size", "set_session", "close", "read"):
        assert callable(getattr(ApexDeviceFIFOQueue, name))
    for name in ("append_to_queue", "sample_batch"):
        assert not hasattr(ApexDeviceFIFOQueue, name)
    for name in ("append", "push", "read", "close", "__len__"):
        assert callable(getattr(DeviceLocalBuffers, name))
    q = _fake_queue()
    q.set_session("s")
    assert q.sess == "s"
    for name in ("drl_apex_queue_create", "drl_apex_queue_destroy", "drl_apex_queue_size", "drl_apex_queue_read",
                 "drl_apex_actor_buffer_create", "drl_apex_actor_buffer_destroy", "drl_apex_actor_buffer_append",
                 "drl_apex_actor_buffer_push", "drl_apex_actor_buffer_size", "drl_apex_actor_buffer_read",
                 "drl_apex_replay_add_from_queue"):
        assert name in native.EXPORTS
