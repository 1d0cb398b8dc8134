"""The device A3C trajectory queue on the GPU: the records A3CVectorActor commits through the A3C recorder against the
records it appends to the host A3CFIFOQueue from the same seeds (bitwise, all six fields, episode ends mid-unroll and
at step T-1, life losses, a reset frame equal to the terminal frame), a3c.Agent.train_from_queue against
a3c.Agent.train of the host copy (bitwise losses, parameters and Adam state, with and without CUDA graphs), the
co-located loop against the host loop, size accounting, blocking and time-outs, step-order errors, reset, an actor
thread beside a learner thread, the plain act after a recorder ran, and the rejections."""
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

T, A = 8, 6
SHAPE = (84, 84, 4)
FIELDS = ("state", "next_state", "previous_action", "action", "reward", "done")


@pytest.fixture(scope="module")
def gpu(native):
    if native.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return native


class SynthEnv:
    """A cheap seeded stand-in for an Atari environment: random frames, rewards in {0, 1, 2}, a life lost now and then
    and episodes of `episode_len` steps.  With same_reset the reset frame is the terminal frame, so the actor's next
    state and the following state are equal bytes across an episode end."""

    def __init__(self, seed, episode_len, same_reset=False):
        self.rng = np.random.RandomState(seed)
        self.episode_len, self.same_reset = episode_len, same_reset
        self.last = None

    def _frame(self):
        return self.rng.randint(0, 256, SHAPE).astype(np.uint8)

    def reset(self):
        self.lives, self.t = 5, 0
        return self.last.copy() if self.same_reset and self.last is not None else self._frame()

    def step(self, a):
        self.t += 1
        if self.rng.rand() < 0.15:
            self.lives -= 1
        self.last = self._frame()
        return self.last, float(self.rng.randint(0, 3)), self.t >= self.episode_len, {"ale.lives": self.lives}


def _envs(n, seed):
    # env 0's first episode ends at step T-1, env 1's reset frame equals its terminal frame, the rest end mid-unroll
    return [SynthEnv(1000 * seed + i, T if i == 0 else 3 + (i % 6), same_reset=(i == 1)) for i in range(n)]


def _policy(graph=True, max_batch=64):
    from distributed_reinforcement_learning_b200.apex_policy import NativeA3CPolicy
    from distributed_reinforcement_learning_b200.model import actor_critic
    p = NativeA3CPolicy(max_batch, num_action=A, input_shape=SHAPE, use_cuda_graph=graph)
    p.set_params(actor_critic.init_params(3, num_action=A, input_shape=SHAPE))
    return p


def _device_queue(n, queue_size=None, trajectory=T, output_size=A):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import A3CDeviceFIFOQueue
    return A3CDeviceFIFOQueue(trajectory, SHAPE, output_size, n, queue_size=queue_size)


class CollectingQueue:
    """An A3CFIFOQueue (capacity 1) drained after every append, as the reference's learner loop drains it; with an
    agent it also trains on each record, as train_a3c.py's learner does."""

    def __init__(self, n, agent=None):
        from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import A3CFIFOQueue
        self.queue, self.agent, self.records, self.losses = A3CFIFOQueue(T, SHAPE, A, n), agent, [], []

    def append_to_queue(self, **kw):
        self.queue.append_to_queue(**kw)
        b = self.queue.sample_batch()
        rec = dict(state=np.stack(b.state[0]), next_state=np.stack(b.next_state[0]),
                   previous_action=np.asarray(b.previous_action[0], np.int32),
                   action=np.asarray(b.action[0], np.int32), reward=np.asarray(b.reward[0], np.float32),
                   done=np.asarray(b.done[0], np.bool_))
        self.records.append(rec)
        if self.agent is not None:
            self.losses.append(self.agent.train(**rec))


def _agent(name, graph):
    from distributed_reinforcement_learning_b200.agent import a3c
    from distributed_reinforcement_learning_b200.model import actor_critic
    ag = a3c.Agent(SHAPE, A, 0.99, 1e-4, 0.0, 1e9, 0.5, 0.01, 40.0, "abs_one", name, name)
    ag.use_cuda_graph = graph
    ag.set_session(None)
    ag._params = actor_critic.init_params(5, num_action=A, input_shape=SHAPE)   # the same start for every agent
    return ag


def _actor(policy, queue, n, seed, learner=None):
    from distributed_reinforcement_learning_b200.actor import A3CVectorActor
    return A3CVectorActor(policy, _envs(n, seed), queue, T, [A - 1] * n, learner=learner)


def _state(agent):
    eng = agent._engine
    return eng.get_params(), eng.get_opt_state()


def _same_state(x, y):
    (px, ox), (py, oy) = x, y
    assert np.array_equal(px, py)
    for k in ox:
        assert np.array_equal(np.asarray(ox[k]), np.asarray(oy[k])), k


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("n", [1, 4, 20])
def test_records_equal_the_host_path(gpu, n, graph):
    unrolls, seed = 3, 7
    np.random.seed(seed)
    host = CollectingQueue(n)
    ah = _actor(_policy(graph), host, n, seed)
    fin_h = [ah.run_unroll() for _ in range(unrolls)]
    rs_h = np.random.get_state()
    np.random.seed(seed)
    dq = _device_queue(n, queue_size=n * unrolls)
    ad = _actor(_policy(graph), dq, n, seed)
    fin_d = [ad.run_unroll() for _ in range(unrolls)]
    rs_d = np.random.get_state()
    assert fin_h == fin_d and any(fin_d)
    assert all(np.array_equal(x, y) for x, y in zip(rs_h, rs_d))
    assert ad.trajs is None and ad.recorder is not None and ah.recorder is None
    assert dq.get_size() == n * unrolls
    ends = lost = 0
    for k, want in enumerate(host.records):
        got = dq.read(k)
        for f in FIELDS:
            assert np.array_equal(got[f], want[f]), (k, f)
        lost += int(want["done"].sum())
    for i in range(n):
        ends += sum(1 for f in fin_d for e in f if e["task"] == i)
    assert ends > 0 and lost > 0
    # env 0's first episode ends at step T-1 of the first unroll
    assert any(e["task"] == 0 and e["episode_step"] == T for e in fin_d[0])


@pytest.mark.parametrize("graph", [True, False])
def test_train_from_queue_is_bitwise_train(gpu, graph):
    n, seed = 3, 5
    np.random.seed(seed)
    dq = _device_queue(n)
    _actor(_policy(), dq, n, seed).run_unroll()
    recs = [dq.read(k) for k in range(n)]
    ah, ad = _agent("a3cq_train_h", graph), _agent("a3cq_train_d", graph)
    for rec in recs:
        lh = ah.train(**rec)
        ld = ad.train_from_queue(dq)
        assert lh == ld
        _same_state(_state(ah), _state(ad))
    assert dq.get_size() == 0


def _loop(agent, queue, unrolls, seed, n, device):
    np.random.seed(seed)
    actor = _actor(_policy(), queue, n, seed, learner=agent)
    losses = []
    for _ in range(unrolls):
        actor.run_unroll()
        if device:
            losses += [agent.train_from_queue(queue) for _ in range(n)]
    return actor, losses


def test_co_located_loop_matches_the_host_loop(gpu):
    n, unrolls, seed = 4, 3, 9
    ah = _agent("a3cq_loop_h", True)
    host = CollectingQueue(n, ah)
    _loop(ah, host, unrolls, seed, n, device=False)
    ad = _agent("a3cq_loop_d", True)
    dq = _device_queue(n)
    _, losses = _loop(ad, dq, unrolls, seed, n, device=True)
    assert len(losses) == n * unrolls and losses == host.losses
    _same_state(_state(ah), _state(ad))


def _unroll(rec, n, seed=0):
    """T acts of random frames with no episode reset (each previous next_state is the next state), -> (frames [T, n],
    the final next_state frames [n])."""
    rng = np.random.RandomState(seed)
    frames = [rng.randint(0, 256, (n,) + SHAPE).astype(np.uint8) for _ in range(T + 1)]
    for t in range(T):
        rec.act(frames[t], np.zeros(n, np.int32), previous_next_state=frames[t] if t else None)
    return frames[:T], frames[T]


def test_size_blocking_timeouts_and_step_order(gpu):
    N = gpu
    n = 2
    pol = _policy()
    dq = _device_queue(n)            # holds n + 1 records
    rec = pol.recorder(dq, n)
    z = np.zeros((n, T))
    st = np.zeros((n,) + SHAPE, np.uint8)
    with pytest.raises(N.DrlError) as ei:
        rec.commit(z, z, st)
    assert ei.value.code == N.DRL_ERR_STATE
    _, last = _unroll(rec, n)
    with pytest.raises(N.DrlError) as ei:
        rec.act(st, np.zeros(n, np.int32), previous_next_state=last)
    assert ei.value.code == N.DRL_ERR_STATE
    rec.commit(z, z, last)
    assert dq.get_size() == n
    _, last = _unroll(rec, n, seed=1)
    with pytest.raises(N.TimeoutError_):
        rec.commit(z, z, last, timeout_ms=0)   # n positions are not free: nothing changes
    assert dq.get_size() == n
    ag = _agent("a3cq_block", True)
    ag.train_from_queue(dq)
    assert dq.get_size() == n - 1
    rec.commit(z, z, last, timeout_ms=0)      # the same unroll, committed once there is room
    assert dq.get_size() == 2 * n - 1
    for _ in range(2 * n - 1):
        ag.train_from_queue(dq)
    slot = ag._slot
    with pytest.raises(N.TimeoutError_):
        ag.train_from_queue(dq, timeout_ms=0)
    assert dq.get_size() == 0 and ag._slot == slot
    # reset after an abandoned unroll: the next unroll starts at step 0 and records only its own steps
    rng = np.random.RandomState(3)
    for _ in range(3):
        f = rng.randint(0, 256, (n,) + SHAPE).astype(np.uint8)
        rec.act(f, np.zeros(n, np.int32), previous_next_state=f)
    rec.reset()
    frames, last = _unroll(rec, n, seed=4)
    rec.commit(z, z, last)
    frames = np.stack(frames)
    for i in range(n):
        r = dq.read(i)
        assert np.array_equal(r["state"], frames[:, i])
        assert np.array_equal(r["next_state"][:-1], frames[1:, i]) and np.array_equal(r["next_state"][-1], last[i])


def test_plain_act_is_unchanged_by_a_recorder(gpu):
    pol = _policy()
    rng = np.random.RandomState(1)
    st = rng.randint(0, 256, (5,) + SHAPE).astype(np.uint8)
    pa = rng.randint(0, A, 5).astype(np.int32)
    u = rng.random_sample(5)
    before = pol.act(st, pa, uniform=u)
    dq = _device_queue(5)
    rec = pol.recorder(dq, 5)
    _, last = _unroll(rec, 5)
    rec.commit(np.zeros((5, T)), np.zeros((5, T)), last)
    after = pol.act(st, pa, uniform=u)
    for k in before:
        assert np.array_equal(before[k], after[k]), k


def test_an_actor_thread_and_a_learner_thread(gpu):
    n, unrolls = 4, 4
    ag = _agent("a3cq_threads", True)
    dq = _device_queue(n)
    actor = _actor(_policy(), dq, n, 21, learner=ag)
    errors, losses = [], []

    def act():
        try:
            for _ in range(unrolls):
                actor.run_unroll()
        except Exception as e:    # pragma: no cover
            errors.append(e)

    def learn():
        try:
            for _ in range(n * unrolls):
                losses.append(ag.train_from_queue(dq, timeout_ms=60000))
        except Exception as e:    # pragma: no cover
            errors.append(e)

    threads = [threading.Thread(target=act), threading.Thread(target=learn)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=300)
    assert not any(t.is_alive() for t in threads) and not errors
    assert len(losses) == n * unrolls and all(np.isfinite(x).all() for x in np.asarray(losses))
    assert dq.get_size() == 0


def test_rejections(gpu):
    import ctypes as C
    N = gpu
    from distributed_reinforcement_learning_b200.a3c_learner import NativeA3CLearner
    from distributed_reinforcement_learning_b200.apex_learner import NativeApexLearner
    from distributed_reinforcement_learning_b200.apex_policy import NativeApexPolicy
    dq = _device_queue(4)
    r = C.c_void_p()
    apol = NativeApexPolicy(8, num_action=A, input_shape=SHAPE)
    assert N.lib.drl_a3c_policy_recorder_create(apol._h, dq._q, 4, C.byref(r)) == N.DRL_ERR_INVALID
    assert "Ape-X" in N.lib.drl_last_error().decode()
    pol = _policy(max_batch=8)
    assert N.lib.drl_a3c_policy_recorder_create(pol._h, dq._q, 9, C.byref(r)) == N.DRL_ERR_INVALID
    assert "max_batch" in N.lib.drl_last_error().decode()
    small = _device_queue(1, queue_size=1)    # at most 2 rows per commit
    assert N.lib.drl_a3c_policy_recorder_create(pol._h, small._q, 3, C.byref(r)) == N.DRL_ERR_INVALID
    assert "never fit" in N.lib.drl_last_error().decode()
    other = _device_queue(4, output_size=A - 1)
    assert N.lib.drl_a3c_policy_recorder_create(pol._h, other._q, 4, C.byref(r)) == N.DRL_ERR_INVALID
    assert "num_action" in N.lib.drl_last_error().decode()
    # learner side: an Ape-X handle, a batch other than T, another num_action
    apex = NativeApexLearner(batch=T, num_action=A)
    assert N.lib.drl_a3c_stage_from_queue(apex._h, 0, dq._q, 0) == N.DRL_ERR_INVALID
    assert "not an A3C handle" in N.lib.drl_last_error().decode()
    lrn = NativeA3CLearner(batch=T + 1, num_action=A)
    with pytest.raises(N.DrlError, match="trajectory"):
        lrn.stage_from_queue(0, dq, 0)
    lrn2 = NativeA3CLearner(batch=T, num_action=A)
    with pytest.raises(N.DrlError, match="num_action"):
        lrn2.stage_from_queue(0, other, 0)
    with pytest.raises(N.DrlError, match="slot"):
        lrn2.stage_from_queue(7, dq, 0)
    # a recorder act without previous_next_state after step 0
    rec = pol.recorder(dq, 4)
    st = np.zeros((4,) + SHAPE, np.uint8)
    rec.act(st, np.zeros(4, np.int32))
    with pytest.raises(N.DrlError, match="previous_next_state"):
        rec.act(st, np.zeros(4, np.int32))
    for h in (rec, pol, apol, apex, lrn, lrn2, dq, small, other):
        h.close()
