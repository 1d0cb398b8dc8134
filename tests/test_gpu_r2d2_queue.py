"""The device R2D2 sequence queue on the GPU: the bytes R2D2VectorActor records through an R2D2 policy recorder against
the records it pushes into the host R2D2FIFOQueue from the same seeds, DeviceMemory.add_from_queue against
DeviceMemory.add of the host batches (bitwise, with and without CUDA graphs), the co-located loop against the host loop,
the recording act against the plain act, size accounting, blocking and time-outs, commit order with two recorders, an
actor thread and a learner thread on one queue, reset and recovery, and the rejections."""
import ctypes as C
import random
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

S, BURN_IN, A, L, B = 15, 7, 4, 64, 16
SHAPE = (84, 84, 1)
FIELDS = ("state", "previous_action", "action", "reward", "done", "previous_h", "previous_c")


@pytest.fixture(scope="module")
def gpu(native):
    if native.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return native


class SynthEnv:
    """A cheap seeded stand-in for an Atari environment: random frames, rewards in {0, 1, 2}, a life lost now and then
    and short episodes, so that unrolls of 15 steps cross life losses and episode ends."""

    def __init__(self, seed):
        self.rng = np.random.RandomState(seed)

    def _frame(self):
        return self.rng.randint(0, 256, SHAPE).astype(np.uint8)

    def reset(self):
        self.lives, self.t = 5, 0
        return self._frame()

    def step(self, a):
        self.t += 1
        if self.rng.rand() < 0.1:
            self.lives -= 1
        done = self.lives == 0 or self.t >= 20 + (a % 5)
        return self._frame(), float(self.rng.randint(0, 3)), done, {"ale.lives": self.lives}


class _RaisingEnv(SynthEnv):
    def __init__(self, seed, fail_at):
        super().__init__(seed)
        self.fail_at, self.calls = fail_at, 0

    def step(self, a):
        self.calls += 1
        if self.calls == self.fail_at:
            raise RuntimeError("environment failed")
        return super().step(a)


def _params(seed=3):
    from distributed_reinforcement_learning_b200.model import r2d2_lstm
    p = r2d2_lstm.init_params(seed, num_action=A, lstm_size=L, input_shape=SHAPE)
    rng = np.random.default_rng(seed + 1)
    return (p + rng.standard_normal(p.shape).astype(np.float32) * 0.01).astype(np.float32)


def _policy(params, max_batch=64, graph=True):
    from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
    p = NativeR2D2Policy(max_batch, num_action=A, lstm_size=L, input_shape=SHAPE, use_cuda_graph=graph)
    p.set_params(params)
    return p


def _device_queue(queue_size=128, batch=B, **kw):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import R2D2DeviceFIFOQueue
    args = dict(seq_len=S, input_shape=SHAPE, output_size=A, queue_size=queue_size, batch_size=batch, num_actors=40,
                lstm_size=L)
    args.update(kw)
    return R2D2DeviceFIFOQueue(**args)


def _host_queue(queue_size=128):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import R2D2FIFOQueue
    return R2D2FIFOQueue(S, SHAPE, A, queue_size, B, 40, L)


def _host_record(q, k):
    """The k-th record of a host R2D2FIFOQueue in R2D2DeviceFIFOQueue.read's form (h, c at step 0)."""
    rec = dict(zip(q._q.fields, q._q._items[k]))
    return dict(state=np.asarray(rec["state"]), previous_action=np.asarray(rec["previous_action"], np.int32),
                action=np.asarray(rec["action"], np.int32), reward=np.asarray(rec["reward"], np.float32),
                done=np.asarray(rec["done"], np.bool_), previous_h=np.asarray(rec["previous_h"][0]),
                previous_c=np.asarray(rec["previous_c"][0]))


def _agent(params, name, graph=True):
    from distributed_reinforcement_learning_b200.agent import r2d2
    from distributed_reinforcement_learning_b200.model import r2d2_lstm
    a = r2d2.Agent(S, BURN_IN, list(SHAPE), A, L, 0.997, 1e-4, 1e-4, 1e9, 40.0, name, name)
    a.use_cuda_graph = graph
    a._main = params.copy()
    a._target = r2d2_lstm.init_params(11, num_action=A, lstm_size=L, input_shape=SHAPE)
    z = np.zeros_like(a._main)
    a._opt = dict(m=z, v=z.copy(), step=0, beta1_power=0.9, beta2_power=0.999)
    return a


def _actor(policy, queue, n, seed, learner=None, epsilon=0.3):
    from distributed_reinforcement_learning_b200.actor import R2D2VectorActor
    actor = R2D2VectorActor(policy, [SynthEnv(1000 * seed + i) for i in range(n)], queue, S, learner=learner)
    actor.epsilon = [epsilon] * n     # some greedy rows, some explore rows
    return actor


def _arms(n, unrolls, seed=11, params=None):
    """Host arm and device arm from the same seeds, parameters and np.random state, `unrolls` unrolls each; checks
    that both finished the same episodes and left np.random in the same state -> (host queue, device queue, device
    actor)."""
    params = _params() if params is None else params
    out = []
    for queue in (_host_queue(), _device_queue()):
        np.random.seed(seed)
        actor = _actor(_policy(params), queue, n, seed)
        fin = [actor.run_unroll() for _ in range(unrolls)]
        out.append((queue, fin, actor, np.random.get_state()[1].copy()))
    (hq, fin_h, ah, rs_h), (dq, fin_d, ad, rs_d) = out
    assert fin_h == fin_d
    assert np.array_equal(rs_h, rs_d)
    assert ad.recorder is not None and ah.recorder is None
    return hq, dq, ad


@pytest.mark.parametrize("n", [1, 16, 20, 40])
def test_recorded_bytes_equal_the_host_path(gpu, n):
    unrolls = 3 if n <= 20 else 2
    hq, dq, _ = _arms(n, unrolls)
    assert hq.get_size() == dq.get_size() == unrolls * n
    saw_life_loss = False
    for k in range(unrolls * n):
        want, got = _host_record(hq, k), dq.read(k)
        for f in FIELDS:
            assert got[f].shape == want[f].shape, (k, f)
            assert np.array_equal(got[f], want[f]), (k, f)
        saw_life_loss |= bool(np.any((got["reward"] == -1.0) & got["done"]))
    assert saw_life_loss
    if n > 1:   # a later unroll starts from the (h, c) carried over, not from zeros
        assert any(dq.read(k)["previous_h"].any() for k in range(n, unrolls * n))


@pytest.mark.parametrize("graph", [True, False])
def test_add_from_queue_is_bitwise_add(gpu, graph):
    params = _params()
    hq, dq, _ = _arms(16, unrolls=3, params=params)
    ag_h, ag_d = _agent(params, "rq_host_%d" % graph, graph), _agent(params, "rq_dev_%d" % graph, graph)
    mem_h, mem_d = ag_h.device_memory(64), ag_d.device_memory(64)
    for _ in range(3):
        b = hq.sample_batch()
        mem_h.add(b.state, b.previous_action, b.action, b.previous_h, b.previous_c, b.reward, b.done)
        mem_d.add_from_queue(dq)
    assert hq.get_size() == dq.get_size() == 0
    assert mem_h.n_entries == mem_d.n_entries == 48
    assert mem_h.total() == mem_d.total()
    rh, rd = mem_h.replay.read(0, 48), mem_d.replay.read(0, 48)
    for k in rh:
        assert np.array_equal(rh[k], rd[k]), k
    u = np.random.RandomState(5).random_sample(B)
    for a, b in zip(mem_h.replay.sample(B, u), mem_d.replay.sample(B, u)):
        assert np.array_equal(a, b)


def _loop(agent, queue, host, iters, seed, n=16, capacity=256):
    """The co-located loop of train_r2d2.py:87-165 with R2D2VectorActor in the same thread."""
    np.random.seed(seed)
    random.seed(seed)
    actor = _actor(_policy(agent._main), queue, n, seed, learner=agent)
    memory = agent.device_memory(capacity)
    out, buffer_step = [], 0
    for _ in range(iters):
        actor.run_unroll()
        if queue.get_size() > B:
            if host:
                b = queue.sample_batch()
                memory.add(b.state, b.previous_action, b.action, b.previous_h, b.previous_c, b.reward, b.done)
            else:
                memory.add_from_queue(queue)
            buffer_step += B
        if buffer_step > 2 * B:
            loss, td = agent.train_from_memory(memory, B)
            out.append((loss, np.array(td), memory.last_sample()[0].copy()))
    return out, memory


def test_co_located_loop_matches_the_host_loop(gpu):
    params = _params()
    ag_h, ag_d = _agent(params, "loop_h"), _agent(params, "loop_d")
    out_h, mem_h = _loop(ag_h, _host_queue(), True, 8, 21)
    out_d, mem_d = _loop(ag_d, _device_queue(), False, 8, 21)
    assert len(out_h) == len(out_d) >= 3
    for (lh, th, ih), (ld, td, idd) in zip(out_h, out_d):
        assert lh == ld and np.isfinite(lh)
        assert np.array_equal(th, td)
        assert np.array_equal(ih, idd)
    assert mem_h.total() == mem_d.total()
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET
    for which in (MAIN, TARGET):
        assert np.array_equal(ag_h._engine.get_params(which), ag_d._engine.get_params(which))


@pytest.mark.parametrize("graph", [True, False])
def test_recording_act_equals_plain_act(gpu, graph):
    params = _params()
    plain, recording = _policy(params, graph=graph), _policy(params, graph=graph)
    dq = _device_queue()
    rec = recording.recorder(dq, 20)
    rng = np.random.RandomState(9)
    for _ in range(2):
        for t in range(S):
            args = (rng.randint(0, 256, (20,) + SHAPE).astype(np.uint8), rng.randint(0, A, 20),
                    rng.randn(20, L).astype(np.float32) * 0.3, rng.randn(20, L).astype(np.float32) * 0.3)
            ex = np.where(rng.rand(20) < 0.3, rng.randint(0, A, 20), -1).astype(np.int32)
            want = plain.act(*args, explore_action=ex)
            got = rec.act(*args, explore_action=ex)
            for k in want:
                assert np.array_equal(want[k], got[k]), (t, k)
            # the plain act graph of the same engine still replays (and for another n) after recording calls
            for n in (20, 7):
                again = recording.act(*[a[:n] for a in args], explore_action=ex[:n])
                ref = plain.act(*[a[:n] for a in args], explore_action=ex[:n])
                for k in ref:
                    assert np.array_equal(ref[k], again[k]), (t, n, k)
            if t == 0:
                first = (args, want)
            if t == 1:
                second = (args, want)
        rec.commit(np.zeros((20, S), np.float32), np.zeros((20, S), np.bool_))
    # row 3 of the second unroll: step 0's h and c, and the frames, previous actions and actions of each step
    got = dq.read(20 + 3)
    (st, pa, h, c), out = first
    assert np.array_equal(got["state"][0], st[3]) and got["previous_action"][0] == pa[3]
    assert np.array_equal(got["previous_h"], h[3]) and np.array_equal(got["previous_c"], c[3])
    assert got["action"][0] == out["action"][3]
    (st, pa, _, _), out = second
    assert np.array_equal(got["state"][1], st[3]) and got["previous_action"][1] == pa[3]
    assert got["action"][1] == out["action"][3]


def _fill(rec, seed):
    """S recorded acts of random inputs on a recorder."""
    rng = np.random.RandomState(seed)
    n = rec.n
    for _ in range(S):
        rec.act(rng.randint(0, 256, (n,) + SHAPE).astype(np.uint8), rng.randint(0, A, n),
                rng.randn(n, L).astype(np.float32) * 0.1, rng.randn(n, L).astype(np.float32) * 0.1,
                explore_action=rng.randint(-1, A, n))


def _commit(rec, seed=0, **kw):
    rng = np.random.RandomState(seed)
    rec.commit(rng.randn(rec.n, S).astype(np.float32), rng.rand(rec.n, S) < 0.1, **kw)


def test_blocking_and_timeouts(gpu):
    N = gpu
    params = _params()
    pol = _policy(params)
    dq = _device_queue(queue_size=16)                    # one slot of 16 plus the spare one
    rec = pol.recorder(dq, 16)
    with pytest.raises(N.DrlError) as ei:
        _commit(rec)
    assert ei.value.code == N.DRL_ERR_STATE and "0 of 15 steps" in str(ei.value)
    for k in range(2):
        _fill(rec, k)
        _commit(rec, k)
    assert dq.get_size() == 32
    first = dq.read(0)
    _fill(rec, 2)
    with pytest.raises(N.DrlError) as ei:
        rec.act(np.zeros((16,) + SHAPE, np.uint8), np.zeros(16, np.int32), np.zeros((16, L), np.float32),
                np.zeros((16, L), np.float32))
    assert ei.value.code == N.DRL_ERR_STATE
    with pytest.raises(N.TimeoutError_):
        _commit(rec, 2, timeout_ms=50)
    assert dq.get_size() == 32
    assert all(np.array_equal(first[f], dq.read(0)[f]) for f in FIELDS)
    ag = _agent(params, "rq_block")
    mem = ag.device_memory(64)
    mem.add_from_queue(dq)
    assert dq.get_size() == 16 and mem.n_entries == 16
    _commit(rec, 2, timeout_ms=5000)                     # the slot the ingest freed
    assert dq.get_size() == 32
    # ingest with fewer than a batch queued
    dq2 = _device_queue()
    rec2 = pol.recorder(dq2, 10)
    _fill(rec2, 5)
    _commit(rec2, 5)
    total = mem.total()
    with pytest.raises(N.TimeoutError_):
        mem.add_from_queue(dq2, timeout_ms=50)
    assert dq2.get_size() == 10 and mem.n_entries == 16 and mem.total() == total
    _fill(rec2, 6)
    _commit(rec2, 6)
    mem.add_from_queue(dq2, timeout_ms=5000)
    assert dq2.get_size() == 4 and mem.n_entries == 32


def test_commit_order_of_two_recorders(gpu):
    params = _params()
    p1, p2 = _policy(params), _policy(params)
    dq = _device_queue()
    r1, r2 = p1.recorder(dq, 20), p2.recorder(dq, 12)

    def fill(rec, tag):
        n = rec.n
        for t in range(S):
            st = np.zeros((n,) + SHAPE, np.uint8)
            st[:, 0, 0, 0] = tag
            st[:, 0, 1, 0] = np.arange(n)
            st[:, 0, 2, 0] = t
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
        assert np.all(got["state"][:, 0, 0, 0] == tag) and np.all(got["state"][:, 0, 1, 0] == row)
        assert np.array_equal(got["state"][:, 0, 2, 0], np.arange(S))
        assert np.all(got["previous_action"] == tag % A)


def test_an_actor_thread_and_a_learner_thread(gpu):
    params = _params()
    dq = _device_queue()
    ag = _agent(params, "rq_threads")
    ag._get_engine(B)
    mem = ag.device_memory(256)
    pol = _policy(params)
    actor = _actor(pol, dq, 16, 5, learner=ag)           # run_unroll syncs the policy under the agent's lock
    unrolls, errors, losses = 8, [], []

    def actor_loop():
        try:
            for _ in range(unrolls):
                actor.run_unroll()
        except Exception as e:    # pragma: no cover - reported below
            errors.append(e)

    def learner_loop():
        try:
            for _ in range(unrolls):
                mem.add_from_queue(dq, timeout_ms=120000)   # waits while the actor thread syncs and records
                losses.append(ag.train_from_memory(mem, B)[0])
        except Exception as e:    # pragma: no cover - reported below
            errors.append(e)

    threads = [threading.Thread(target=actor_loop), threading.Thread(target=learner_loop)]
    for th in threads:
        th.start()
    for th in threads:
        th.join(timeout=300)
    assert not any(th.is_alive() for th in threads), "deadlock"
    assert not errors, errors
    assert len(losses) == unrolls and np.isfinite(losses).all()
    assert mem.n_entries == unrolls * 16 and dq.get_size() == 0


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
    assert ei.value.code == N.DRL_ERR_STATE and "7 of 15 steps" in str(ei.value)
    rec.reset()
    _fill(rec, 9)                                        # a whole unroll from step 0
    _commit(rec, 9)
    rng = np.random.RandomState(9)
    want_state = rng.randint(0, 256, (8,) + SHAPE).astype(np.uint8)
    rng.randint(0, A, 8)
    want_h = rng.randn(8, L).astype(np.float32) * 0.1
    got = dq.read(0)
    assert dq.get_size() == 8 and np.array_equal(got["state"][0], want_state[0])
    assert np.array_equal(got["previous_h"], want_h[0])


def test_vector_actor_recovers_after_an_environment_raises(gpu):
    pol = _policy(_params())
    dq = _device_queue()
    from distributed_reinforcement_learning_b200.actor import R2D2VectorActor
    actor = R2D2VectorActor(pol, [SynthEnv(5), _RaisingEnv(6, fail_at=9)], dq, S)
    with pytest.raises(RuntimeError, match="environment failed"):
        actor.run_unroll()
    assert dq.get_size() == 0
    actor.run_unroll()                                   # starts again at step 0 and commits a whole unroll
    actor.run_unroll()
    assert dq.get_size() == 4
    assert all(dq.read(k)["state"].shape == (S,) + SHAPE for k in range(4))


def test_closing_the_policy_closes_its_recorders(gpu):
    pol = _policy(_params())
    dq = _device_queue()
    rec = pol.recorder(dq, 8)
    _fill(rec, 1)
    _commit(rec, 1)
    pol.close()                      # what the garbage collector may do first when both are garbage
    assert not rec._r.value
    rec.close()
    assert dq.get_size() == 8 and dq.read(7)["state"].shape == (S,) + SHAPE


def test_rejections(gpu):
    N = gpu
    from distributed_reinforcement_learning_b200.r2d2_learner import NativeR2D2Learner
    params = _params()
    pol = _policy(params, max_batch=16)
    ag = _agent(params, "rq_reject")
    learner = ag._get_engine(B)
    mem = ag.device_memory(64)
    if N.device_count() < 2:
        with pytest.raises(N.DrlError, match="no CPU fallback"):
            _device_queue(device=N.device_count())
    else:
        q1 = _device_queue(device=1)
        with pytest.raises(N.DrlError, match="device"):
            pol.recorder(q1, 8)
        with pytest.raises(N.DrlError, match="device"):
            mem.replay.add_from_queue(learner, q1, 10)
    for kw, what in ((dict(seq_len=10), "seq_len"), (dict(output_size=6), "num_action"),
                     (dict(input_shape=(84, 84, 4)), "channels")):
        q = _device_queue(**kw)
        with pytest.raises(N.DrlError, match=what) as ei:
            mem.replay.add_from_queue(learner, q, 10)
        assert ei.value.code == N.DRL_ERR_INVALID
        assert q.get_size() == 0
        if what != "seq_len":
            with pytest.raises(N.DrlError, match="num_action" if what == "num_action" else "frames"):
                pol.recorder(q, 8)
    big = _device_queue(batch=32)
    with pytest.raises(N.DrlError, match="exceeds the learner's batch"):
        mem.replay.add_from_queue(learner, big, 10)
    small_learner = NativeR2D2Learner(batch=8, seq_len=S, burn_in=BURN_IN, num_action=A, lstm_size=L,
                                      input_shape=SHAPE)
    with pytest.raises(N.DrlError, match="exceeds the learner's batch"):
        mem.replay.add_from_queue(small_learner, _device_queue(), 10)
    small_learner.close()
    q = _device_queue()
    with pytest.raises(ValueError, match="n = 20"):
        pol.recorder(q, 20)
    r = C.c_void_p()
    assert N.lib.drl_r2d2_policy_recorder_create(pol._h, q._q, 20, C.byref(r)) == N.DRL_ERR_INVALID
    assert "max_batch" in N.lib.drl_last_error().decode()
    tiny = _device_queue(queue_size=8, batch=8)          # 2 slots of 8: at most 9 rows per commit
    with pytest.raises(N.DrlError, match="never fit"):
        pol.recorder(tiny, 12)
    # the recorder checks previous and explore actions at act time, as the plain act does
    rec = pol.recorder(q, 4)
    z = np.zeros((4, L), np.float32)
    st = np.zeros((4,) + SHAPE, np.uint8)
    for pa, ex in ((np.array([0, 1, 2, 4]), None), (np.zeros(4, np.int32), np.array([-1, 0, 4, 1]))):
        rc = N.lib.drl_r2d2_policy_recorder_act(rec._r, N.ptr(st), N.ptr(pa.astype(np.int32)), N.ptr(z), N.ptr(z),
                                                N.ptr(ex.astype(np.int32)) if ex is not None else None,
                                                None, None, None, None, None)
        assert rc == N.DRL_ERR_INVALID and "outside" in N.lib.drl_last_error().decode()
    _fill(rec, 3)                                        # nothing was recorded by the refused acts
    _commit(rec, 3)
    assert q.get_size() == 4
