"""CPU (no GPU needed): the device A3C trajectory queue and the A3C recorder refuse to run without a device (no CPU
fallback), their argument checks that come before any device work, A3CVectorActor's refusal of a device queue that
does not fit its policy, a3c.Agent.train_from_queue's checks and its wait without the agent's lock, and the surface of
the new Python API."""
import ctypes as C
import threading

import numpy as np
import pytest

T, A, NA = 32, 6, 20
SHAPE = (84, 84, 4)


def _fake_queue(**kw):
    """An A3CDeviceFIFOQueue's attributes without a device handle (the checks under test run before any device work)."""
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import A3CDeviceFIFOQueue
    q = A3CDeviceFIFOQueue.__new__(A3CDeviceFIFOQueue)
    q.trajectory, q.input_shape, q.output_size = T, SHAPE, A
    q.num_actors, q.queue_size, q.max_rows, q.device = NA, NA, NA + 1, 0
    q._q = C.c_void_p()
    for k, v in kw.items():
        setattr(q, k, v)
    return q


def _fake_policy(**kw):
    from distributed_reinforcement_learning_b200.apex_policy import NativeA3CPolicy
    p = NativeA3CPolicy.__new__(NativeA3CPolicy)
    p.max_batch, p.A, p.input_shape, p.device = 64, A, SHAPE, 0
    p._h = C.c_void_p()
    for k, v in kw.items():
        setattr(p, k, v)
    return p


class _Env:
    def reset(self):
        return np.zeros(SHAPE, np.uint8)


def _agent(name="host_a3cq"):
    from distributed_reinforcement_learning_b200.agent import a3c
    return a3c.Agent(input_shape=SHAPE, num_action=A, discount_factor=0.99, start_learning_rate=1e-4,
                     end_learning_rate=0.0, learning_frame=1e9, baseline_loss_coef=0.5, entropy_coef=0.01,
                     gradient_clip_norm=40.0, reward_clipping="abs_one", model_name=name, learner_name=name)


def test_creation_fails_loudly_without_a_device(native):
    if native.device_count() > 0:
        pytest.skip("a CUDA device is present")
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import A3CDeviceFIFOQueue
    with pytest.raises(native.DrlError) as ei:
        A3CDeviceFIFOQueue(T, SHAPE, A, NA)
    assert "no CPU fallback" in str(ei.value) and ei.value.code == native.DRL_ERR_CUDA
    r = C.c_void_p()
    assert native.lib.drl_a3c_policy_recorder_create(None, None, 1, C.byref(r)) == native.DRL_ERR_CUDA
    assert "no CPU fallback" in native.lib.drl_last_error().decode()


def test_arguments_are_checked_before_looking_for_a_device(native):
    N = native
    q = C.c_void_p()
    for args, what in (((0, A, 4, 0), "trajectory"), ((513, A, 4, 0), "trajectory"), ((T, 1, 4, 0), "num_action"),
                       ((T, 33, 4, 0), "num_action"), ((T, A, 0, 0), "capacity"), ((T, A, 4, 99), "no CPU fallback")):
        rc = N.lib.drl_a3c_queue_create(*args, C.byref(q))
        assert rc == (N.DRL_ERR_CUDA if what == "no CPU fallback" else N.DRL_ERR_INVALID), args
        err = N.lib.drl_last_error().decode()
        assert what in err
        if what != "no CPU fallback":
            assert err.startswith("a3c queue")
    assert N.lib.drl_a3c_queue_create(T, A, 4, 0, None) == N.DRL_ERR_INVALID
    assert N.lib.drl_a3c_policy_recorder_create(None, None, 1, None) == N.DRL_ERR_INVALID
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import A3CDeviceFIFOQueue
    with pytest.raises(ValueError, match="input_shape"):
        A3CDeviceFIFOQueue(T, (84, 84, 1), A, NA)


def test_entry_points_reject_null_handles(native):
    N = native
    z = np.zeros(SHAPE, np.uint8)
    assert N.lib.drl_a3c_queue_destroy(None) == N.DRL_OK
    assert N.lib.drl_a3c_queue_size(None) == 0
    assert N.lib.drl_a3c_queue_read(None, 0, *[N.ptr(z)] * 6) == N.DRL_ERR_INVALID
    assert "null a3c queue handle" in N.lib.drl_last_error().decode()
    assert N.lib.drl_a3c_policy_recorder_destroy(None) == N.DRL_OK
    for call in (lambda: N.lib.drl_a3c_policy_recorder_act(None, *[N.ptr(z)] * 7),
                 lambda: N.lib.drl_a3c_policy_recorder_commit(None, N.ptr(z), N.ptr(z), N.ptr(z), -1),
                 lambda: N.lib.drl_a3c_policy_recorder_reset(None)):
        assert call() == N.DRL_ERR_INVALID
        assert "null recorder handle" in N.lib.drl_last_error().decode()
    assert N.lib.drl_a3c_stage_from_queue(None, 0, None, -1) == N.DRL_ERR_INVALID


def test_recorder_python_side_validation(native):
    from distributed_reinforcement_learning_b200.apex_policy import A3CPolicyRecorder, NativeApexPolicy
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import (ApexDeviceFIFOQueue,
                                                                                         DeviceFIFOQueue)
    p = _fake_policy()
    with pytest.raises(TypeError, match="A3CDeviceFIFOQueue"):
        p.recorder(ApexDeviceFIFOQueue.__new__(ApexDeviceFIFOQueue), 4)
    with pytest.raises(TypeError, match="A3CDeviceFIFOQueue"):
        p.recorder(DeviceFIFOQueue.__new__(DeviceFIFOQueue), 4)
    with pytest.raises(ValueError, match="n = 65"):
        p.recorder(_fake_queue(), 65)
    assert not hasattr(NativeApexPolicy, "recorder")
    r = A3CPolicyRecorder.__new__(A3CPolicyRecorder)
    r.policy, r.queue, r.n, r.T, r._r = p, _fake_queue(), 4, T, C.c_void_p()
    st = np.zeros((4,) + SHAPE, np.uint8)
    pa = np.zeros(4, np.int32)
    with pytest.raises(ValueError, match="recorder act: 3 rows"):
        r.act(st[:3], pa[:3], uniform=np.zeros(3))
    with pytest.raises(ValueError, match="uniform: values"):
        r.act(st, pa, uniform=np.ones(4))
    with pytest.raises(ValueError, match="previous_next_state: expected shape"):
        r.act(st, pa, uniform=np.zeros(4), previous_next_state=st[:2])
    with pytest.raises(ValueError, match="reward: expected shape"):
        r.commit(np.zeros((4, T - 1)), np.zeros((4, T)), st)
    with pytest.raises(ValueError, match="next_state: expected shape"):
        r.commit(np.zeros((4, T)), np.zeros((4, T)), st[:, :80])


@pytest.mark.parametrize("kw,what", [(dict(trajectory=16), "unrolls of 16"), (dict(output_size=4), "num_action"),
                                     (dict(device=1), "device"), (dict(max_rows=8), "at most 8")])
def test_vector_actor_rejects_a_device_queue_that_does_not_fit(native, kw, what):
    from distributed_reinforcement_learning_b200.actor import A3CVectorActor
    with pytest.raises(ValueError, match=what):
        A3CVectorActor(_fake_policy(), [_Env() for _ in range(NA)], _fake_queue(**kw), T, [A] * NA)


def test_train_from_queue_python_side_validation(native, monkeypatch):
    from distributed_reinforcement_learning_b200 import dp
    from distributed_reinforcement_learning_b200.a3c_learner import NativeA3CLearner
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import ApexDeviceFIFOQueue
    eng = NativeA3CLearner.__new__(NativeA3CLearner)
    eng._h, eng._keep = C.c_void_p(), {}
    with pytest.raises(TypeError, match="A3CDeviceFIFOQueue"):
        eng.stage_from_queue(0, object())
    with pytest.raises(TypeError, match="A3CDeviceFIFOQueue"):
        eng.stage_from_queue(0, ApexDeviceFIFOQueue.__new__(ApexDeviceFIFOQueue))
    monkeypatch.setattr(dp, "distributed", lambda: True)
    with pytest.raises(RuntimeError, match="single-replica"):
        _agent().train_from_queue(_fake_queue())


class _SpyEngine:
    B, num_slots = T, 2

    def __init__(self, agent, fail=False):
        self.agent, self.fail, self.held, self.staged = agent, fail, [], []

    def stage_from_queue(self, slot, queue, timeout_ms):
        def other_thread():
            got = self.agent._lock.acquire(timeout=1.0)
            self.held.append(got)
            if got:
                self.agent._lock.release()
        t = threading.Thread(target=other_thread)
        t.start()
        t.join()
        if self.fail:
            raise TimeoutError("queue empty")
        self.staged.append((slot, queue, timeout_ms))

    def step(self, slot):
        return dict(pi_loss=1.0, baseline_loss=2.0, entropy=3.0, learning_rate=4.0, slot=slot)


def test_train_from_queue_waits_without_the_agents_lock(native):
    """The pop blocks inside the C call; actor threads take the agent's lock in sync_policy meanwhile."""
    ag = _agent("host_a3cq_lock")
    ag._ensure_init()
    eng = _SpyEngine(ag)
    ag._engine = eng
    q = _fake_queue()
    assert ag.train_from_queue(q, timeout_ms=7) == (1.0, 2.0, 3.0, 4.0)
    assert eng.held == [True] and eng.staged == [(0, q, 7)] and ag._last["slot"] == 0
    assert ag._slot == 1
    # a failed wait gives the slot back
    eng.fail = True
    with pytest.raises(TimeoutError):
        ag.train_from_queue(q, timeout_ms=0)
    assert eng.held == [True, True] and ag._slot == 1


def test_surface(native):
    from distributed_reinforcement_learning_b200.a3c_learner import NativeA3CLearner
    from distributed_reinforcement_learning_b200.agent import a3c
    from distributed_reinforcement_learning_b200.apex_policy import A3CPolicyRecorder, NativeA3CPolicy
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import A3CDeviceFIFOQueue
    assert callable(a3c.Agent.train_from_queue)
    assert callable(NativeA3CLearner.stage_from_queue)
    assert callable(NativeA3CPolicy.recorder)
    for name in ("act", "commit", "reset", "close"):
        assert callable(getattr(A3CPolicyRecorder, name))
    for name in ("get_size", "set_session", "close", "read"):
        assert callable(getattr(A3CDeviceFIFOQueue, name))
    for name in ("append_to_queue", "sample_batch"):
        assert not hasattr(A3CDeviceFIFOQueue, name)
    q = _fake_queue()
    q.set_session("s")
    assert q.sess == "s"
    for name in ("drl_a3c_queue_create", "drl_a3c_queue_destroy", "drl_a3c_queue_size", "drl_a3c_queue_read",
                 "drl_a3c_policy_recorder_create", "drl_a3c_policy_recorder_destroy", "drl_a3c_policy_recorder_act",
                 "drl_a3c_policy_recorder_commit", "drl_a3c_policy_recorder_reset", "drl_a3c_stage_from_queue"):
        assert name in native.EXPORTS
