"""The device IMPALA trajectory queue on the GPU: the bytes VectorActor records through a policy recorder against the
bytes it pushes into the host ring from the same seeds, learner steps from the queue against steps on the host
batches (bitwise, with and without CUDA graphs), size accounting, blocking and time-outs, commit order with several
recorders, two actor threads and a learner thread on one queue, the rejections, and the unchanged plain act path."""
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

T, A, L, B = 20, 18, 256, 32
SHAPE = (84, 84, 4)
FIELDS = ("state", "reward", "done", "behavior_policy", "action", "previous_action", "previous_h", "previous_c")


@pytest.fixture(scope="module")
def gpu(native):
    if native.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return native


class SynthEnv:
    """A cheap seeded stand-in for an Atari environment: random frames, rewards in {0, 1, 2}, a life lost now and then
    and short episodes, so that unrolls of 20 steps cross life losses and episode ends."""

    def __init__(self, seed):
        self.rng = np.random.RandomState(seed)

    def _frame(self):
        return self.rng.randint(0, 256, SHAPE).astype(np.uint8)

    def reset(self):
        self.lives, self.t = 5, 0
        return self._frame()

    def step(self, a):
        self.t += 1
        if self.rng.rand() < 0.15:
            self.lives -= 1
        done = self.lives == 0 or self.t >= 25 + (a % 7)
        return self._frame(), float(self.rng.randint(0, 3)), done, {"ale.lives": self.lives}


def _params(seed=7):
    from distributed_reinforcement_learning_b200.model import impala_actor_critic
    p = impala_actor_critic.init_params(seed=seed, num_action=A, lstm_hidden_size=L, input_shape=SHAPE)
    rng = np.random.default_rng(seed + 1)
    return (p + rng.standard_normal(p.shape).astype(np.float32) * 0.01).astype(np.float32)


def _policy(params, max_batch=64, graph=True):
    from distributed_reinforcement_learning_b200.policy import NativePolicy
    p = NativePolicy(max_batch, num_action=A, use_cuda_graph=graph)
    p.set_params(params)
    return p


def _device_queue(queue_size=128, batch=B, **kw):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import DeviceFIFOQueue
    args = dict(trajectory=T, input_shape=SHAPE, output_size=A, queue_size=queue_size, batch_size=batch, num_actors=20,
                lstm_size=L)
    args.update(kw)
    return DeviceFIFOQueue(**args)


def _host_queue():
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import FIFOQueue

    class LoggingFIFOQueue(FIFOQueue):
        """The ring, plus a log of every trajectory pushed, in push (= FIFO) order."""
        log = None

        def append_to_queue(self, **kw):
            if self.log is None:
                self.log = []
            self.log.append({k: np.array(v) for k, v in kw.items()})
            super().append_to_queue(**kw)

    return LoggingFIFOQueue(T, SHAPE, A, 128, B, 20, L)


def _agent(params, name, graph=True):
    from distributed_reinforcement_learning_b200.agent import impala
    ag = impala.Agent(trajectory=T, input_shape=SHAPE, num_action=A, lstm_hidden_size=L, discount_factor=0.99,
                      start_learning_rate=0.0006, end_learning_rate=0.0, learning_frame=1e9, baseline_loss_coef=1.0,
                      entropy_coef=0.05, gradient_clip_norm=40.0, reward_clipping="abs_one", model_name=name,
                      learner_name=name)
    ag.use_cuda_graph = graph
    ag._ensure_init()
    ag._params = params.copy()
    return ag


def _arms(n, unrolls, seed=11, params=None):
    """Host arm and device arm from the same seeds, parameters and np.random state, `unrolls` unrolls each; checks
    that both finished the same episodes and left np.random in the same state -> (hq, dq, host actor, device actor)."""
    from distributed_reinforcement_learning_b200.actor import VectorActor
    params = _params() if params is None else params
    out = []
    for queue in (_host_queue(), _device_queue()):
        np.random.seed(seed)
        pol = _policy(params)
        actor = VectorActor(pol, [SynthEnv(1000 * seed + i) for i in range(n)], queue, T, [A] * n)
        fin = [actor.run_unroll() for _ in range(unrolls)]
        out.append((queue, fin, actor, np.random.get_state()[1].copy()))
    (hq, fin_h, ah, rs_h), (dq, fin_d, ad, rs_d) = out
    assert fin_h == fin_d
    assert np.array_equal(rs_h, rs_d)
    return hq, dq, ah, ad


def _host_traj(entry):
    return dict(state=entry["unrolled_state"], reward=entry["unrolled_reward"].astype(np.float32),
                done=entry["unrolled_done"].astype(np.bool_), behavior_policy=entry["unrolled_behavior_policy"],
                action=entry["unrolled_action"].astype(np.int32),
                previous_action=entry["unrolled_previous_action"].astype(np.int32),
                previous_h=entry["unrolled_previous_h"], previous_c=entry["unrolled_previous_c"])


@pytest.mark.parametrize("n", [20, 32])
def test_recorded_bytes_equal_the_host_ring(gpu, n):
    hq, dq, ah, ad = _arms(n, unrolls=3)
    assert hq.get_size() == dq.get_size() == 3 * n
    assert ad.recorder is not None and ah.recorder is None
    saw_life_loss = saw_reset = False
    for k in range(3 * n):
        want = _host_traj(hq.log[k])
        got = dq.read(k)
        for f in FIELDS:
            assert got[f].dtype == want[f].dtype or f == "done", f
            assert np.array_equal(got[f], want[f]), (k, f)
        saw_life_loss |= bool(np.any((got["reward"] == -1.0) & got["done"]))
        t_after_end = np.nonzero(got["done"][:-1])[0] + 1
        saw_reset |= any(not got["previous_h"][t].any() and got["previous_action"][t] == 0 for t in t_after_end)
    assert saw_life_loss and saw_reset
    # the ring's own first batch, row for row
    batch = hq.sample_batch()
    for k in range(B):
        got = dq.read(k)
        for f, v in zip(("state", "reward", "done", "behavior_policy", "action", "previous_action", "previous_h",
                         "previous_c"),
                        (batch.state, batch.reward, batch.done, batch.behavior_policy, batch.action,
                         batch.previous_action, batch.previous_h, batch.previous_c)):
            assert np.array_equal(got[f], np.asarray(v[k])), (k, f)


@pytest.mark.parametrize("graph", [True, False])
def test_train_from_queue_is_bitwise_train(gpu, graph):
    params = _params()
    hq, dq, _, _ = _arms(32, unrolls=3, params=params)
    ag_h, ag_d = _agent(params, "q_host_%d" % graph, graph), _agent(params, "q_dev_%d" % graph, graph)
    for _ in range(3):
        b = hq.sample_batch()
        rh = ag_h.train(b.state, b.reward, b.action, b.done, b.behavior_policy, b.previous_action, b.previous_h,
                        b.previous_c)
        rd = ag_d.train_from_queue(dq)
        assert rh == rd
        assert ag_h._last == ag_d._last
        assert np.isfinite(rd).all()
    assert dq.get_size() == hq.get_size() == 0
    assert np.array_equal(ag_h._engine.get_params(), ag_d._engine.get_params())


def _fill(rec, seed):
    """T recorded acts of random inputs on a recorder."""
    rng = np.random.RandomState(seed)
    n = rec.n
    for _ in range(T):
        rec.act(rng.randint(0, 256, (n,) + SHAPE).astype(np.uint8), rng.randint(0, A, n),
                rng.randn(n, L).astype(np.float32) * 0.1, rng.randn(n, L).astype(np.float32) * 0.1,
                uniform=rng.random_sample(n))


def _commit(rec, seed=0, **kw):
    rng = np.random.RandomState(seed)
    rec.commit(rng.randn(rec.n, T).astype(np.float32), rng.rand(rec.n, T) < 0.1, **kw)


def test_size_tracks_the_host_queue(gpu):
    from distributed_reinforcement_learning_b200.actor import VectorActor
    params = _params()
    hq, dq = _host_queue(), _device_queue()
    ag_h, ag_d = _agent(params, "size_h"), _agent(params, "size_d")
    actors = []
    for q in (hq, dq):
        np.random.seed(3)
        actors.append(VectorActor(_policy(params), [SynthEnv(50 + i) for i in range(20)], q, T, [A] * 20))
    for it in range(6):
        for act in actors:
            np.random.seed(100 + it)
            act.run_unroll()
        assert hq.get_size() == dq.get_size()
        while hq.get_size() > B:
            b = hq.sample_batch()
            ag_h.train(b.state, b.reward, b.action, b.done, b.behavior_policy, b.previous_action, b.previous_h,
                       b.previous_c)
            ag_d.train_from_queue(dq)
            assert hq.get_size() == dq.get_size()


def test_blocking_and_timeouts(gpu):
    N = gpu
    params = _params()
    pol = _policy(params)
    # a full queue: capacity 32 = one slot of 32 plus the spare one
    dq = _device_queue(queue_size=32)
    rec = pol.recorder(dq, 32)
    with pytest.raises(N.DrlError) as ei:
        _commit(rec)
    assert ei.value.code == N.DRL_ERR_STATE and "0 of 20 steps" in str(ei.value)
    for k in range(2):
        _fill(rec, k)
        _commit(rec, k)
    assert dq.get_size() == 64
    first = dq.read(0)
    _fill(rec, 2)
    with pytest.raises(N.DrlError) as ei:
        rec.act(np.zeros((32,) + SHAPE, np.uint8), np.zeros(32, np.int32), np.zeros((32, L), np.float32),
                np.zeros((32, L), np.float32))
    assert ei.value.code == N.DRL_ERR_STATE
    with pytest.raises(N.TimeoutError_):
        _commit(rec, 2, timeout_ms=50)
    assert dq.get_size() == 64
    assert all(np.array_equal(first[f], dq.read(0)[f]) for f in FIELDS)
    ag = _agent(params, "block")
    ag.train_from_queue(dq)
    assert dq.get_size() == 32
    _commit(rec, 2, timeout_ms=5000)     # the slot the learner freed
    assert dq.get_size() == 64
    # staging with fewer than a batch queued
    dq2 = _device_queue()
    rec2 = pol.recorder(dq2, 20)
    _fill(rec2, 5)
    _commit(rec2, 5)
    slot = ag._slot
    with pytest.raises(N.TimeoutError_):
        ag.train_from_queue(dq2, timeout_ms=50)
    assert dq2.get_size() == 20 and ag._slot == slot
    _fill(rec2, 6)
    _commit(rec2, 6)
    ag.train_from_queue(dq2, timeout_ms=5000)
    assert dq2.get_size() == 8 and ag._slot != slot


def test_commit_order_of_two_recorders(gpu):
    params = _params()
    p1, p2 = _policy(params), _policy(params)
    dq = _device_queue()
    r1, r2 = p1.recorder(dq, 20), p2.recorder(dq, 12)

    def fill(rec, tag):
        n = rec.n
        for t in range(T):
            st = np.zeros((n,) + SHAPE, np.uint8)
            st[:, 0, 0, 0] = tag
            st[:, 0, 0, 1] = np.arange(n)
            st[:, 0, 0, 2] = t
            rec.act(st, np.full(n, tag % A), np.zeros((n, L), np.float32), np.zeros((n, L), np.float32))

    fill(r1, 1)
    fill(r2, 2)
    _commit(r2)
    _commit(r1)
    fill(r1, 3)
    _commit(r1)
    want = [(2, i) for i in range(12)] + [(1, i) for i in range(20)] + [(3, i) for i in range(20)]
    assert dq.get_size() == len(want)
    for k, (tag, row) in enumerate(want):
        got = dq.read(k)
        assert np.all(got["state"][:, 0, 0, 0] == tag) and np.all(got["state"][:, 0, 0, 1] == row)
        assert np.array_equal(got["state"][:, 0, 0, 2], np.arange(T))
        assert np.all(got["previous_action"] == tag % A)


def test_two_actor_threads_and_a_learner_thread(gpu):
    from distributed_reinforcement_learning_b200.actor import VectorActor
    params = _params()
    dq = _device_queue()
    ag = _agent(params, "threads")
    pols = [_policy(params), _policy(params)]
    actors = [VectorActor(pols[j], [SynthEnv(700 + 16 * j + i) for i in range(16)], dq, T, [A] * 16)
              for j in range(2)]
    unrolls, errors, losses = 6, [], []
    n_train = 2 * unrolls * 16 // B

    def actor_loop(a):
        try:
            for _ in range(unrolls):
                a.run_unroll()
        except Exception as e:    # pragma: no cover - reported below
            errors.append(e)

    def learner_loop():
        try:
            for _ in range(n_train):
                losses.append(ag.train_from_queue(dq, timeout_ms=120000))
                for p in pols:
                    ag.sync_policy(p)
        except Exception as e:    # pragma: no cover - reported below
            errors.append(e)

    threads = [threading.Thread(target=actor_loop, args=(a,)) for a in actors] + [threading.Thread(target=learner_loop)]
    for th in threads:
        th.start()
    for th in threads:
        th.join(timeout=300)
    assert not any(th.is_alive() for th in threads), "deadlock"
    assert not errors, errors
    committed = 2 * unrolls * 16
    assert committed == len(losses) * B + dq.get_size()
    assert np.isfinite(np.array(losses)).all()


def test_rejections(gpu):
    import ctypes as C
    N = gpu
    from distributed_reinforcement_learning_b200.learner import NativeLearner
    params = _params()
    pol = _policy(params, max_batch=16)
    learner = NativeLearner(batch=B, trajectory=T, num_action=A)
    if N.device_count() < 2:
        with pytest.raises(N.DrlError, match="no CPU fallback"):
            _device_queue(device=N.device_count())
    else:
        q1 = _device_queue(device=1)
        with pytest.raises(N.DrlError, match="device"):
            pol.recorder(q1, 8)
        with pytest.raises(N.DrlError, match="device"):
            learner.stage_from_queue(0, q1, 10)
    for kw, what in ((dict(trajectory=10), "trajectory"), (dict(output_size=6), "num_action"),
                     (dict(batch=16), "batch"), (dict(input_shape=(84, 84, 1)), "frames")):
        q = _device_queue(**kw)
        with pytest.raises(N.DrlError, match=what) as ei:
            learner.stage_from_queue(0, q, 10)
        assert ei.value.code == N.DRL_ERR_INVALID
        assert q.get_size() == 0
        if what in ("num_action", "frames"):
            with pytest.raises(N.DrlError, match=what):
                pol.recorder(q, 8)
    q = _device_queue()
    with pytest.raises(ValueError, match="n = 20"):
        pol.recorder(q, 20)
    r = C.c_void_p()
    assert N.lib.drl_policy_recorder_create(pol._h, q._q, 20, C.byref(r)) == N.DRL_ERR_INVALID
    assert "max_batch" in N.lib.drl_last_error().decode()
    small = _device_queue(queue_size=32)          # 2 slots of 32: at most 33 rows per commit
    with pytest.raises(N.DrlError, match="never fit"):
        _policy(params).recorder(small, 40)
    with pytest.raises(N.DrlError, match="slot 5 out of range"):
        learner.stage_from_queue(5, q, 10)


@pytest.mark.parametrize("graph", [True, False])
def test_recording_engine_acts_like_a_plain_one(gpu, graph):
    params = _params()
    plain, recording = _policy(params, graph=graph), _policy(params, graph=graph)
    dq = _device_queue()
    rec = recording.recorder(dq, 20)
    rng = np.random.RandomState(9)
    for _ in range(2):
        for t in range(T):
            args = (rng.randint(0, 256, (20,) + SHAPE).astype(np.uint8), rng.randint(0, A, 20),
                    rng.randn(20, L).astype(np.float32) * 0.1, rng.randn(20, L).astype(np.float32) * 0.1)
            u = rng.random_sample(20)
            want = plain.act(*args, uniform=u)
            got = rec.act(*args, uniform=u)
            for k in want:
                assert np.array_equal(want[k], got[k]), (t, k)
            # the plain act graph of the same engine still replays (and for another n) after recording calls
            for n in (20, 7):
                again = recording.act(*[a[:n] for a in args], uniform=u[:n])
                ref = plain.act(*[a[:n] for a in args], uniform=u[:n])
                for k in ref:
                    assert np.array_equal(ref[k], again[k]), (t, n, k)
            if t == 0:
                first = (args, want)
        _commit(rec)
    # the recorded step 0 of row 3 of the second unroll is what act was given and returned
    got = dq.read(20 + 3)
    (st, pa, h, c), out = first
    assert np.array_equal(got["state"][0], st[3]) and got["previous_action"][0] == pa[3]
    assert np.array_equal(got["previous_h"][0], h[3]) and np.array_equal(got["previous_c"][0], c[3])
    assert np.array_equal(got["behavior_policy"][0], out["policy"][3]) and got["action"][0] == out["action"][3]


def test_closing_the_policy_closes_its_recorders(gpu):
    pol = _policy(_params())
    dq = _device_queue()
    rec = pol.recorder(dq, 8)
    _fill(rec, 1)
    _commit(rec, 1)
    pol.close()                      # what the garbage collector may do first when both are garbage
    assert not rec._r.value
    rec.close()
    assert dq.get_size() == 8 and dq.read(7)["state"].shape == (T,) + SHAPE


def test_reset_discards_an_abandoned_unroll(gpu):
    N = gpu
    pol = _policy(_params())
    dq = _device_queue()
    rec = pol.recorder(dq, 8)
    rng = np.random.RandomState(4)
    for _ in range(7):                                   # an unroll abandoned after 7 steps
        rec.act(rng.randint(0, 256, (8,) + SHAPE).astype(np.uint8), np.zeros(8, np.int32),
                np.zeros((8, L), np.float32), np.zeros((8, L), np.float32))
    with pytest.raises(N.DrlError) as ei:
        _commit(rec)
    assert ei.value.code == N.DRL_ERR_STATE and "7 of 20 steps" in str(ei.value)
    rec.reset()
    _fill(rec, 9)                                        # a whole unroll from step 0
    _commit(rec, 9)
    want = np.random.RandomState(9).randint(0, 256, (8,) + SHAPE).astype(np.uint8)
    assert dq.get_size() == 8 and np.array_equal(dq.read(0)["state"][0], want[0])


class _RaisingEnv(SynthEnv):
    def __init__(self, seed, fail_at):
        super().__init__(seed)
        self.fail_at, self.calls = fail_at, 0

    def step(self, a):
        self.calls += 1
        if self.calls == self.fail_at:
            raise RuntimeError("environment failed")
        return super().step(a)


def test_vector_actor_recovers_after_an_environment_raises(gpu):
    from distributed_reinforcement_learning_b200.actor import VectorActor
    pol = _policy(_params())
    dq = _device_queue()
    envs = [SynthEnv(5)] + [_RaisingEnv(6, fail_at=9)]
    actor = VectorActor(pol, envs, dq, T, [A] * 2)
    with pytest.raises(RuntimeError, match="environment failed"):
        actor.run_unroll()
    assert dq.get_size() == 0
    actor.run_unroll()                                   # starts again at step 0 and commits a whole unroll
    actor.run_unroll()
    assert dq.get_size() == 4
    assert all(dq.read(k)["state"].shape == (T,) + SHAPE for k in range(4))


def test_train_from_queue_takes_its_slot_before_waiting(gpu):
    N = gpu
    params = _params()
    pol = _policy(params)
    dq = _device_queue()
    ag = _agent(params, "slot")
    rec = pol.recorder(dq, 32)
    seen = []
    real = ag._get_engine(B).stage_from_queue

    def spy(slot, queue, timeout_ms=-1):
        seen.append((slot, ag._slot))                    # the slot staged, and what a train() meanwhile would take
        return real(slot, queue, timeout_ms)

    ag._engine.stage_from_queue = spy
    with pytest.raises(N.TimeoutError_):
        ag.train_from_queue(dq, timeout_ms=20)
    assert ag._slot == 0 and seen == [(0, 1)]
    for k in range(2):
        _fill(rec, k)
        _commit(rec, k)
        ag.train_from_queue(dq)
    assert seen[1:] == [(0, 1), (1, 0)] and ag._slot == 0
