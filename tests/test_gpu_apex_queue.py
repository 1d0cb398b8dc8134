"""The device Ape-X transition queue and actor buffers on the GPU: the records ApexVectorActor pushes through
DeviceLocalBuffers against the records it pushes into the host ApexFIFOQueue from the same seeds (bitwise, with rings
that wrap and evict), DeviceMemory.add_from_queue against DeviceMemory.add of the host records (bitwise, with and
without CUDA graphs), the co-located loop against the host loop, size accounting, blocking and time-outs, an actor
thread beside a learner thread, closing, and the rejections."""
import random
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

T, A, B = 8, 6, 16
SHAPE = (84, 84, 4)
CAP = 4 * T + 5                       # every ring wraps and evicts within 6 unrolls (48 appends)
FIELDS = ("state", "next_state", "previous_action", "action", "reward", "done")


@pytest.fixture(scope="module")
def gpu(native):
    if native.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return native


class SynthEnv:
    """A cheap seeded stand-in for an Atari environment: random frames, rewards in {0, 1, 2}, a life lost now and then
    and short episodes, so that unrolls cross life losses and episode ends."""

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
        done = self.lives == 0 or self.t >= 12 + (a % 5)
        return self._frame(), float(self.rng.randint(0, 3)), done, {"ale.lives": self.lives}


def _params(seed=3):
    from distributed_reinforcement_learning_b200.model import apex_value
    return apex_value.init_params(seed, num_action=A, input_shape=SHAPE)


def _policy(params, graph=True):
    from distributed_reinforcement_learning_b200.apex_policy import NativeApexPolicy
    p = NativeApexPolicy(64, num_action=A, input_shape=SHAPE, use_cuda_graph=graph)
    p.set_params(params)
    return p


def _device_queue(queue_size=1024, trajectory=T, output_size=A, **kw):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import ApexDeviceFIFOQueue
    return ApexDeviceFIFOQueue(trajectory, SHAPE, output_size, queue_size, B, 20, **kw)


def _host_queue(queue_size=1024):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import ApexFIFOQueue
    return ApexFIFOQueue(T, SHAPE, A, queue_size, B, 20)


def _host_record(q, k):
    """The k-th record of a host ApexFIFOQueue in ApexDeviceFIFOQueue.read's form."""
    rec = dict(zip(q._q.fields, q._q._items[k]))
    return dict(state=np.stack(rec["state"]), next_state=np.stack(rec["next_state"]),
                previous_action=np.asarray(rec["previous_action"], np.int32),
                action=np.asarray(rec["action"], np.int32), reward=np.asarray(rec["reward"], np.float32),
                done=np.asarray(rec["done"], np.bool_))


def _agent(params, name, graph=True):
    from distributed_reinforcement_learning_b200.agent import apex
    from distributed_reinforcement_learning_b200.model import apex_value
    a = apex.Agent(SHAPE, A, 0.99, 40.0, "abs_one", 1e-4, 0.0, 1e9, name, name)
    a.use_cuda_graph = graph
    a._main = params.copy()
    a._target = apex_value.init_params(11, num_action=A, input_shape=SHAPE)
    z = np.zeros_like(a._main)
    a._opt = dict(m=z, v=z.copy(), step=0, beta1_power=0.9, beta2_power=0.999)
    return a


def _actor(policy, queue, n, seed, learner=None, epsilon=0.3):
    from distributed_reinforcement_learning_b200.actor import ApexVectorActor
    actor = ApexVectorActor(policy, [SynthEnv(1000 * seed + i) for i in range(n)], queue, T, [A - 1] * n,
                            learner=learner, buffer_capacity=CAP)
    actor.epsilon = [epsilon] * n     # some greedy rows, some explore rows
    return actor


def _arms(n, unrolls, seed=11, params=None):
    """Host arm and device arm from the same seeds, parameters and np.random state, `unrolls` unrolls each; checks
    that both finished the same episodes and left np.random in the same state -> (host queue, device queue, host
    actor, device actor)."""
    params = _params() if params is None else params
    out = []
    for queue in (_host_queue(), _device_queue()):
        np.random.seed(seed)
        actor = _actor(_policy(params), queue, n, seed)
        fin = [actor.run_unroll() for _ in range(unrolls)]
        out.append((queue, fin, actor, np.random.get_state()))
    (hq, fin_h, ah, rs_h), (dq, fin_d, ad, rs_d) = out
    assert fin_h == fin_d and any(fin_d)     # episodes ended: their next states were uploaded, not copied
    assert all(np.array_equal(x, y) for x, y in zip(rs_h, rs_d))
    assert ad.device_buffers is not None and ah.device_buffers is None
    return hq, dq, ah, ad


@pytest.mark.parametrize("n", [1, 4, 20])
def test_records_equal_the_host_path(gpu, n):
    unrolls = 6
    hq, dq, ah, ad = _arms(n, unrolls)
    pushes = n * (unrolls * T - 3 * T)           # every step once a buffer holds more than 3T transitions
    assert hq.get_size() == dq.get_size() == pushes
    saw_life_loss = False
    for k in range(pushes):
        want, got = _host_record(hq, k), dq.read(k)
        for f in FIELDS:
            assert got[f].shape == want[f].shape, (k, f)
            assert np.array_equal(got[f], want[f]), (k, f)
        saw_life_loss |= bool(np.any((got["reward"] == -1.0) & got["done"]))
    assert saw_life_loss
    # the deques themselves, after the rings wrapped
    db = ad.device_buffers
    assert len(db) == len(ah.buffers[0]) == CAP
    for i in range(n):
        hb = ah.buffers[i]
        for j in range(CAP):
            got = db.read(i, j)
            assert np.array_equal(got["state"], hb.state[j]) and np.array_equal(got["next_state"], hb.next_state[j])
            assert (got["previous_action"], got["action"]) == (hb.previous_action[j], hb.action[j])
            assert got["reward"] == np.float32(hb.reward[j]) and got["done"] == bool(hb.done[j])


@pytest.mark.parametrize("graph", [True, False])
def test_add_from_queue_is_bitwise_add(gpu, graph):
    params = _params()
    hq, dq, _, _ = _arms(4, unrolls=4, params=params)
    assert hq.get_size() == dq.get_size() == 32
    ag_h, ag_d = _agent(params, "aq_host_%d" % graph, graph), _agent(params, "aq_dev_%d" % graph, graph)
    mem_h, mem_d = ag_h.device_memory(200), ag_d.device_memory(200)
    for _ in range(30):                           # 240 transitions: the memories wrap too
        b = hq.sample_batch(1)
        mem_h.add(b.state[0], b.next_state[0], b.previous_action[0], b.action[0], b.reward[0], b.done[0])
        mem_d.add_from_queue(dq)
    assert hq.get_size() == dq.get_size() == 2
    assert mem_h.n_entries == mem_d.n_entries == 200
    assert mem_h.total() == mem_d.total()
    rh, rd = mem_h.replay.read(0, 200), mem_d.replay.read(0, 200)
    for k in rh:
        assert np.array_equal(rh[k], rd[k]), k
    u = np.random.RandomState(5).random_sample(B)
    for a, b in zip(mem_h.replay.sample(B, u), mem_d.replay.sample(B, u)):
        assert np.array_equal(a, b)


def _loop(agent, queue, host, iters, seed, n=4):
    """The co-located loop of train_apex.py:82-231 in one thread: an actor unroll, the ingest of every queued record,
    then one training step once more than 10 records were ingested."""
    np.random.seed(seed)
    random.seed(seed)
    actor = _actor(_policy(agent._main), queue, n, seed, learner=agent)
    memory = agent.device_memory(512)
    out, buffer_step = [], 0
    for _ in range(iters):
        actor.run_unroll()
        while queue.get_size():
            if host:
                b = queue.sample_batch(1)
                memory.add(b.state[0], b.next_state[0], b.previous_action[0], b.action[0], b.reward[0], b.done[0])
            else:
                memory.add_from_queue(queue)
            buffer_step += 1
        if buffer_step > 10:
            loss, td = agent.train_from_memory(memory, B)
            out.append((loss, np.array(td), memory.last_sample()[0].copy()))
    return out, memory


def test_co_located_loop_matches_the_host_loop(gpu):
    params = _params()
    ag_h, ag_d = _agent(params, "aloop_h"), _agent(params, "aloop_d")
    out_h, mem_h = _loop(ag_h, _host_queue(), True, 8, 21)
    out_d, mem_d = _loop(ag_d, _device_queue(), False, 8, 21)
    assert len(out_h) == len(out_d) >= 3
    for (lh, th, ih), (ld, td, idd) in zip(out_h, out_d):
        assert lh == ld and np.isfinite(lh)
        assert np.array_equal(th, td)
        assert np.array_equal(ih, idd)
    assert mem_h.total() == mem_d.total()
    from distributed_reinforcement_learning_b200.apex_learner import MAIN, TARGET
    for which in (MAIN, TARGET):
        assert np.array_equal(ag_h._engine.get_params(which), ag_d._engine.get_params(which))


def _buffers(n=2, capacity=40, fill=3 * T + 1, seed=0):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import DeviceLocalBuffers
    db = DeviceLocalBuffers(n, capacity, A)
    rng = np.random.RandomState(seed)
    for _ in range(fill):
        db.append(rng.randint(0, 256, (n,) + SHAPE).astype(np.uint8), rng.randint(0, 256, (n,) + SHAPE).astype(np.uint8),
                  rng.randint(0, A, n), rng.randint(0, A, n), rng.randn(n), rng.rand(n) < 0.1)
    return db


def test_size_blocking_and_timeouts(gpu):
    N = gpu
    db = _buffers()
    assert len(db) == 3 * T + 1
    dq = _device_queue(queue_size=2)              # 2 + 1 slots
    for k in range(3):
        db.push(dq, k % 2, np.arange(T) + k)
        assert dq.get_size() == k + 1
    first = dq.read(0)
    with pytest.raises(N.TimeoutError_):
        db.push(dq, 0, np.arange(T), timeout_ms=50)
    assert dq.get_size() == 3
    assert all(np.array_equal(first[f], dq.read(0)[f]) for f in FIELDS)
    got = db.read(0, 0)
    assert np.array_equal(first["state"][0], got["state"]) and first["previous_action"][0] == got["previous_action"]
    ag = _agent(_params(), "aq_block")
    mem = ag.device_memory(64)
    mem.add_from_queue(dq)
    assert dq.get_size() == 2 and mem.n_entries == T
    db.push(dq, 1, np.arange(T), timeout_ms=5000)  # the slot the ingest freed
    assert dq.get_size() == 3
    for _ in range(3):
        mem.add_from_queue(dq, timeout_ms=5000)
    total = mem.total()
    with pytest.raises(N.TimeoutError_):
        mem.add_from_queue(dq, timeout_ms=50)
    assert dq.get_size() == 0 and mem.n_entries == 4 * T and mem.total() == total
    with pytest.raises(N.DrlError, match="outside"):
        dq.read(0)


def test_an_actor_thread_and_a_learner_thread(gpu):
    params = _params()
    dq = _device_queue(queue_size=16)
    ag = _agent(params, "aq_threads")
    ag._get_engine(B)
    mem = ag.device_memory(512)
    n, unrolls = 4, 6
    actor = _actor(_policy(params), dq, n, 5, learner=ag)   # run_unroll syncs the policy under the agent's lock
    records = n * (unrolls * T - 3 * T)
    errors, losses = [], []

    def actor_loop():
        try:
            for _ in range(unrolls):
                actor.run_unroll()
        except Exception as e:    # pragma: no cover - reported below
            errors.append(e)

    def learner_loop():
        try:
            for k in range(records):
                mem.add_from_queue(dq, timeout_ms=120000)   # waits while the actor thread syncs and pushes
                if k % 8 == 7:
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
    assert len(losses) == records // 8 and np.isfinite(losses).all()
    assert mem.n_entries == min(records * T, 512) and dq.get_size() == 0


def test_closing(gpu):
    db = _buffers()
    dq = _device_queue(queue_size=4)
    for k in range(3):
        db.push(dq, 0, np.arange(T))
    dq.close()                                    # waits for the pushes' gathers
    assert not dq._q.value and dq.get_size() == 0
    dq.close()
    assert len(db) == 3 * T + 1
    db.close()
    assert not db._b.value
    db.close()


def test_rejections(gpu):
    N = gpu
    from distributed_reinforcement_learning_b200.a3c_learner import NativeA3CLearner
    from distributed_reinforcement_learning_b200.apex_learner import NativeApexLearner
    params = _params()
    ag = _agent(params, "aq_reject")
    learner = ag._get_engine(B)
    mem = ag.device_memory(64)
    db = _buffers()
    if N.device_count() < 2:
        with pytest.raises(N.DrlError, match="no CPU fallback"):
            _device_queue(device=N.device_count())
    else:
        q1 = _device_queue(device=1)
        with pytest.raises(N.DrlError, match="device"):
            db.push(q1, 0, np.arange(T))
        with pytest.raises(N.DrlError, match="device"):
            mem.replay.add_from_queue(learner, q1, 10)
    q_a = _device_queue(output_size=4)
    with pytest.raises(N.DrlError, match="num_action") as ei:
        db.push(q_a, 0, np.arange(T))
    assert ei.value.code == N.DRL_ERR_INVALID and q_a.get_size() == 0
    with pytest.raises(N.DrlError, match="num_action"):
        mem.replay.add_from_queue(learner, q_a, 10)
    big = _device_queue(trajectory=B + 1)
    with pytest.raises(N.DrlError, match="exceeds the learner's batch"):
        mem.replay.add_from_queue(learner, big, 10)
    small = NativeApexLearner(batch=T - 1, num_action=A, input_shape=SHAPE)
    with pytest.raises(N.DrlError, match="exceeds the learner's batch"):
        mem.replay.add_from_queue(small, _device_queue(), 10)
    small.close()
    a3c = NativeA3CLearner(batch=B, num_action=A, input_shape=SHAPE)
    with pytest.raises(N.DrlError, match="A3C"):
        mem.replay.add_from_queue(a3c, _device_queue(), 10)
    a3c.close()
    # the native checks behind the Python ones: actions at append, deque indices at push, nothing changed
    q = _device_queue()
    n, length = db.n, len(db)
    st = np.zeros((n,) + SHAPE, np.uint8)
    z = np.zeros(n, np.float32)
    u8 = np.zeros(n, np.uint8)
    for pa, ac in ((np.array([0, A], np.int32), np.zeros(n, np.int32)), (np.zeros(n, np.int32), np.array([-1, 0], np.int32))):
        rc = N.lib.drl_apex_actor_buffer_append(db._b, n, N.ptr(st), N.ptr(st), N.ptr(pa), N.ptr(ac), N.ptr(z), N.ptr(u8))
        assert rc == N.DRL_ERR_INVALID and "not in [0, %d)" % A in N.lib.drl_last_error().decode()
    rc = N.lib.drl_apex_actor_buffer_append(db._b, n + 1, N.ptr(st), N.ptr(st), N.ptr(u8), N.ptr(u8), N.ptr(z), N.ptr(u8))
    assert rc == N.DRL_ERR_INVALID and "environments" in N.lib.drl_last_error().decode()
    assert len(db) == length
    for order in (np.arange(T, dtype=np.int32) + length - T + 1, np.arange(T, dtype=np.int32) - 1):
        rc = N.lib.drl_apex_actor_buffer_push(db._b, q._q, 0, N.ptr(order), 10)
        assert rc == N.DRL_ERR_INVALID and "outside" in N.lib.drl_last_error().decode()
    rc = N.lib.drl_apex_actor_buffer_push(db._b, q._q, n, N.ptr(np.arange(T, dtype=np.int32)), 10)
    assert rc == N.DRL_ERR_INVALID and "env" in N.lib.drl_last_error().decode()
    assert q.get_size() == 0
    db.push(q, 0, np.arange(T) + length - T)      # the newest T transitions: accepted
    assert q.get_size() == 1
    got, want = q.read(0), db.read(0, length - 1)
    assert np.array_equal(got["next_state"][T - 1], want["next_state"]) and got["action"][T - 1] == want["action"]
