"""The A3C policy server on the GPU (drl_a3c_policy_server_*, actor_server.py: A3CEnvWorkerPool, A3CPolicyServer): the
A3C engine's batch-composition invariance it rests on, the unrolls it commits against a serial n = 1 oracle that
follows the A3C actor's rules (next_state included), the queue's backpressure on the workers, an end-to-end run beside a
training learner, the engine's plain act after a server ran on it, and the argument checks."""
import ctypes as C
import functools
import mmap
import multiprocessing as mp
import threading
import time

import numpy as np
import pytest

T, A = 8, 4
SHAPE = (84, 84, 4)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def N(native):
    if native.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return native


class SynthEnv:
    """A cheap seeded stand-in for an Atari environment: random frames, rewards in {0, 1, 2}, a life lost now and then,
    and episodes of `length` steps (or until the lives run out), so that unrolls cross life losses and episode ends."""

    def __init__(self, seed, length):
        self.rng, self.length = np.random.RandomState(seed), length

    def _frame(self):
        return self.rng.randint(0, 256, SHAPE).astype(np.uint8)

    def reset(self):
        self.lives, self.t = 5, 0
        return self._frame()

    def step(self, a):
        self.t += 1
        if self.rng.rand() < 0.15:
            self.lives -= 1
        done = self.lives == 0 or self.t >= self.length
        return self._frame(), float(self.rng.randint(0, 3)), done, {"ale.lives": self.lives}


def _length(i):
    # environment 0 ends its first episode at step T-1 of the first unroll, the others mid-unroll or across unrolls
    return T if i == 0 else 3 + (5 * i) % 11


def _params(seed=7, num_action=A):
    from distributed_reinforcement_learning_b200.model import actor_critic
    p = actor_critic.init_params(seed, num_action=num_action, input_shape=SHAPE)
    rng = np.random.default_rng(seed + 1)
    return (p + rng.standard_normal(p.shape).astype(np.float32) * 0.01).astype(np.float32)


def _policy(params, max_batch=64, graph=True, num_action=A):
    from distributed_reinforcement_learning_b200.apex_policy import NativeA3CPolicy
    p = NativeA3CPolicy(max_batch, num_action=num_action, input_shape=SHAPE, use_cuda_graph=graph)
    p.set_params(params)
    return p


def _queue(queue_size, trajectory=T, num_action=A):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import A3CDeviceFIFOQueue
    return A3CDeviceFIFOQueue(trajectory, SHAPE, num_action, 1, queue_size=queue_size)


def _pool(num_envs, per_worker, seed0=100):
    from distributed_reinforcement_learning_b200.actor_server import A3CEnvWorkerPool
    return A3CEnvWorkerPool([functools.partial(SynthEnv, seed0 + i, _length(i)) for i in range(num_envs)],
                            [A] * num_envs, per_worker, seeds=[seed0 + 1000 + i for i in range(num_envs)])


def _agent(name):
    from distributed_reinforcement_learning_b200.agent import a3c
    ag = a3c.Agent(SHAPE, A, 0.99, 1e-4, 0.0, 1e9, 0.5, 0.01, 40.0, "abs_one", name, name)
    ag.use_cuda_graph = True
    ag.set_session(None)
    ag._params = _params(5)
    return ag


def _no_children():
    deadline = time.time() + 15
    while mp.active_children() and time.time() < deadline:
        time.sleep(0.05)
    return not mp.active_children()


def _serve_lockstep(server, pool, rounds, rng, max_chunk):
    """`rounds` steps of every environment: wait for every worker, serve all environments in random order and random
    chunk sizes, answer the workers."""
    for _ in range(rounds):
        ready = []
        while len(ready) < pool.num_workers:
            ready, _ = pool.wait_ready(120)
        ids = rng.permutation(pool.num_envs).astype(np.int32)
        k = 0
        while k < len(ids):
            c = int(rng.randint(1, max_chunk + 1))
            server.serve(ids[k:k + c])
            k += c
        pool.reply(ready)


def test_act_is_invariant_to_batch_composition(N):
    """A row's policy, action and max_prob do not depend on the other rows of its batch or on its position, for n =
    1..64: the server serves any subset of environments in any order, and its bit-equality with the n = 1 oracle rests
    on this."""
    pol = _policy(_params())
    try:
        rng = np.random.RandomState(3)
        n = 64
        st = rng.randint(0, 256, (n,) + SHAPE).astype(np.uint8)
        pa = rng.randint(0, A, n).astype(np.int32)
        u = rng.random_sample(n)
        full = pol.act(st, pa, uniform=u)

        def same(out, i, r):
            for k in ("policy", "action", "max_prob"):
                assert np.array_equal(out[k][i], full[k][r]), (k, i, r)

        for r in (0, 63, 17):
            same(pol.act(st[r:r + 1], pa[r:r + 1], uniform=u[r:r + 1]), 0, r)
        for pos in (0, 63):
            idx = np.insert(np.array([i for i in range(n) if i != 5][:63]), pos, 5)
            out = pol.act(st[idx], pa[idx], uniform=u[idx])
            for i, r in enumerate(idx):
                same(out, i, r)
        for m in range(1, n + 1):
            idx = rng.permutation(n)[:m]
            out = pol.act(st[idx], pa[idx], uniform=u[idx])
            for i, r in enumerate(idx):
                same(out, i, r)
    finally:
        pol.close()


def _oracle(pol, seed0, num_envs, unrolls):
    """Per task: its own env and RandomState, NativeA3CPolicy.act at n = 1, the A3C actor's rules
    (utils.impala_env_step).  -> (the records of `unrolls` unrolls of every task as the queue stores them, the
    (task, unroll, step) of every episode end, the number of life losses)."""
    from distributed_reinforcement_learning_b200 import utils
    from distributed_reinforcement_learning_b200.actor_server import _Stats
    out, ends, lives_lost = [], [], 0
    for i in range(num_envs):
        env, rs = SynthEnv(seed0 + i, _length(i)), np.random.RandomState(seed0 + 1000 + i)
        stats = _Stats(1)
        state, pa = env.reset(), 0
        for u in range(unrolls):
            tr = {k: [] for k in ("state", "next_state", "previous_action", "action", "reward", "done")}
            for t in range(T):
                o = pol.act(state[None], np.array([pa], np.int32), uniform=np.array([rs.random_sample()]))
                a = int(o["action"][0])
                next_state, r, d, new_state, ep = utils.impala_env_step(env, a, A, stats, 0, o["max_prob"][0])
                lives_lost += ep is None and d
                for k, v in (("state", state), ("next_state", next_state), ("previous_action", pa), ("action", a),
                             ("reward", r), ("done", d)):
                    tr[k].append(v)
                if ep is not None:
                    ends.append((i, u, t))
                state, pa = new_state, (0 if ep is not None else a)
            out.append(dict(state=np.stack(tr["state"]), next_state=np.stack(tr["next_state"]),
                            previous_action=np.array(tr["previous_action"], np.int32),
                            action=np.array(tr["action"], np.int32), reward=np.array(tr["reward"], np.float32),
                            done=np.array(tr["done"], np.bool_)))
    return out, ends, lives_lost


@pytest.mark.parametrize("graph", [True, False], ids=["graph", "eager"])
def test_served_unrolls_match_serial_oracle(N, graph):
    from distributed_reinforcement_learning_b200.actor_server import A3CPolicyServer
    P, k, U = 3, 4, 3
    E = P * k
    params = _params(11)
    pol = _policy(params, max_batch=8, graph=graph)
    q = _queue(E * U)
    pool = _pool(E, k)
    server = None
    try:
        server = A3CPolicyServer(pol, q, pool)
        # U unrolls and the reports carrying the last one's final rewards and next_state frames
        _serve_lockstep(server, pool, U * T + 1, np.random.RandomState(5), 8)
        assert q.get_size() == E * U
        got = [q.read(j) for j in range(E * U)]
    finally:
        if server is not None:
            server.close()
        pool.close()
    oracle_pol = _policy(params, max_batch=1, graph=graph)
    try:
        want, ends, lives_lost = _oracle(oracle_pol, 100, E, U)
    finally:
        oracle_pol.close()
    q.close()
    pol.close()
    # the data crosses episode ends mid-unroll and at step T-1, and life losses
    assert any(t == T - 1 for _, _, t in ends) and any(t < T - 1 for _, _, t in ends) and lives_lost > 0
    by_frames = {w["state"].tobytes(): w for w in want}
    assert len(by_frames) == len(want)
    matched = set()
    for g in got:
        key = g["state"].tobytes()
        assert key in by_frames and key not in matched
        matched.add(key)
        w = by_frames[key]
        assert set(g) == set(w)
        for f in w:
            assert g[f].dtype == w[f].dtype and np.array_equal(g[f].view(np.uint8), w[f].view(np.uint8)), f
    assert len(matched) == len(want)
    assert _no_children()


def test_full_queue_blocks_serve_until_the_learner_pops(N):
    from distributed_reinforcement_learning_b200.actor_server import A3CPolicyServer
    Ts, E = 5, 4
    q = _queue(2 * E - 1, trajectory=Ts)     # 2E records: two unrolls of every environment fit
    ag = _agent("a3c_server_bp")
    pol = _policy(_params(2), max_batch=4)
    pool = _pool(E, 2, seed0=300)
    server = None
    try:
        server = A3CPolicyServer(pol, q, pool)
        rng = np.random.RandomState(1)
        _serve_lockstep(server, pool, 2 * Ts + 1, rng, 4)
        assert q.get_size() == 2 * E
        _serve_lockstep(server, pool, Ts - 1, rng, 4)     # the third unroll up to its last step
        ready = []
        while len(ready) < pool.num_workers:
            ready, _ = pool.wait_ready(120)
        pool.views["action"][:] = -7
        ids = np.arange(E, dtype=np.int32)
        t0 = time.time()
        with pytest.raises(N.TimeoutError_):
            server.serve(ids, timeout_ms=300)
        assert time.time() - t0 >= 0.25
        assert q.get_size() == 2 * E and (pool.views["action"][:E] == -7).all()   # nothing changed
        for _ in range(E):
            losses = ag.train_from_queue(q)
            assert np.isfinite(losses).all()
        assert q.get_size() == E
        server.serve(ids, timeout_ms=10000)
        pool.reply(ready)
        assert q.get_size() == 2 * E and (pool.views["action"][:E] >= 0).all()
        for _ in range(2 * E):
            ag.train_from_queue(q)
        assert q.get_size() == 0   # 3 unrolls of 4 environments committed, 12 records trained on
    finally:
        if server is not None:
            server.close()
        pool.close()
        pol.close()
        q.close()
    assert _no_children()


def test_end_to_end_with_training_learner(N):
    from distributed_reinforcement_learning_b200.actor_server import A3CPolicyServer
    steps = 6
    ag = _agent("a3c_server_e2e")
    ag._get_engine(T)
    before = ag._engine.get_params()
    q = _queue(32)
    pol = _policy(_params(9))
    pool = _pool(24, 2, seed0=500)
    assert pool.num_workers == 12
    server = A3CPolicyServer(pol, q, pool, learner=ag)
    stop, losses, errors, episodes = threading.Event(), [], [], []

    def serve():
        try:
            server.run(stop, on_episodes=episodes.extend)
        except Exception as e:   # pragma: no cover - reported below
            errors.append(e)

    th = threading.Thread(target=serve)
    th.start()
    try:
        for _ in range(steps):
            losses.append(ag.train_from_queue(q, timeout_ms=120000))
    finally:
        stop.set()
        th.join(60)
        server.close()
        pool.close()
    assert not th.is_alive() and not errors
    assert np.isfinite(np.array(losses)).all()
    assert not np.array_equal(ag._engine.get_params(), before)
    assert server.syncs >= 2 and sum(server.batch_sizes.values()) > 0
    assert all(set(e) == {"task", "episode", "prob", "score", "episode_step"} for e in episodes)
    pol.close()
    q.close()
    assert _no_children()


def test_plain_act_unchanged_after_a_server_ran(N):
    """The server runs the engine's forward half on its own input rows and outputs; the plain act's staging, outputs
    and graphs are the engine's, so NativeA3CPolicy.act gives the same results before and after."""
    from distributed_reinforcement_learning_b200.actor_server import A3CPolicyServer
    pol = _policy(_params(6), max_batch=4)
    rng = np.random.RandomState(8)
    st = rng.randint(0, 256, (3,) + SHAPE).astype(np.uint8)
    pa = rng.randint(0, A, 3).astype(np.int32)
    u = rng.random_sample(3)
    before = pol.act(st, pa, uniform=u)
    q = _queue(8, trajectory=3)
    pool = _pool(3, 3, seed0=900)
    try:
        server = A3CPolicyServer(pol, q, pool)
        _serve_lockstep(server, pool, 7, np.random.RandomState(2), 3)
        server.close()
        after = pol.act(st, pa, uniform=u)
    finally:
        pool.close()
        q.close()
        pol.close()
    for k in ("policy", "action", "max_prob"):
        assert np.array_equal(before[k], after[k]), k
    assert _no_children()


class _Block:
    """An exchange block without workers: page-aligned anonymous memory (A3C-sized unless `size` says otherwise)."""

    def __init__(self, num_envs, size=None, offset=0):
        from distributed_reinforcement_learning_b200.actor_server import a3c_exchange_bytes
        self.num_envs = num_envs
        self.exchange_bytes = a3c_exchange_bytes(num_envs) if size is None else size
        self._m = mmap.mmap(-1, max(a3c_exchange_bytes(num_envs), self.exchange_bytes) + mmap.PAGESIZE)
        self._anchor = C.c_char.from_buffer(self._m)
        self.address = C.addressof(self._anchor) + offset


def _create(N, pol, q, blk):
    s = C.c_void_p()
    rc = N.lib.drl_a3c_policy_server_create(pol._h, q._q, blk.num_envs, C.c_void_p(blk.address), blk.exchange_bytes,
                                            C.byref(s))
    if rc == 0:
        N.lib.drl_a3c_policy_server_destroy(s)
    return rc


def test_exchange_bytes_entry_point(N):
    from distributed_reinforcement_learning_b200.actor_server import a3c_exchange_bytes
    b = C.c_int64()
    for n in (1, 7, 256):
        N.check(N.lib.drl_a3c_policy_server_exchange_bytes(n, C.byref(b)))
        assert b.value == a3c_exchange_bytes(n)
    for n in (0, 257):
        assert N.lib.drl_a3c_policy_server_exchange_bytes(n, C.byref(b)) == N.DRL_ERR_INVALID


def test_argument_checks_and_reregistration(N):
    from distributed_reinforcement_learning_b200.actor_server import A3CPolicyServer, exchange_bytes
    from distributed_reinforcement_learning_b200.apex_policy import NativeApexPolicy
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import DeviceFIFOQueue
    pol = _policy(_params(1), max_batch=4)
    q = _queue(8)
    blk = _Block(6)
    apex = NativeApexPolicy(4, num_action=A, input_shape=SHAPE)
    try:
        # an Ape-X engine (the C-ABI accepts its handle type; the server refuses algo 0), and the other queue type
        assert _create(N, apex, q, blk) == N.DRL_ERR_INVALID
        assert "algo 1" in N.lib.drl_last_error().decode()
        with pytest.raises(TypeError, match="NativeA3CPolicy"):
            A3CPolicyServer(apex, q, blk)
        other_type = DeviceFIFOQueue(T, SHAPE, A, 8, 4, 1, 256)
        with pytest.raises(TypeError, match="A3CDeviceFIFOQueue"):
            A3CPolicyServer(pol, other_type, blk)
        other_type.close()
        other = _queue(8, num_action=A + 1)
        with pytest.raises(N.DrlError, match="num_action"):
            A3CPolicyServer(pol, other, blk)
        other.close()
        # an IMPALA-sized block, a misaligned one, one byte short, too many environments
        for bad in (_Block(6, size=exchange_bytes(6)), _Block(6, offset=16),
                    _Block(6, size=_Block(6).exchange_bytes - 1)):
            assert _create(N, pol, q, bad) == N.DRL_ERR_INVALID
        assert _create(N, pol, q, _Block(257, size=1 << 26)) == N.DRL_ERR_INVALID
        assert _create(N, pol, q, _Block(0, size=4096)) == N.DRL_ERR_INVALID
        # a queue that cannot take min(num_envs, max_batch) = 4 records at once
        small = _queue(2)
        with pytest.raises(N.DrlError, match="at once"):
            A3CPolicyServer(pol, small, blk)
        small.close()
        server = A3CPolicyServer(pol, q, blk)
        for ids in ([6], [-1], [0, 2, 0], [0, 1, 2, 3, 4]):
            with pytest.raises(N.DrlError) as e:
                server.serve(ids)
            assert e.value.code == N.DRL_ERR_INVALID
        server.close()
        with pytest.raises(ValueError, match="closed"):
            server.serve([0])
        # the block was unregistered: it can be registered again
        server = A3CPolicyServer(pol, q, blk)
        server.close()
    finally:
        apex.close()
        pol.close()
        q.close()


def test_closing_the_pool_closes_its_server(N):
    """The pool frees the exchange block only after its server has unregistered it."""
    from distributed_reinforcement_learning_b200.actor_server import A3CPolicyServer
    pol = _policy(_params(1), max_batch=4)
    q = _queue(8)
    pool = _pool(2, 1, seed0=700)
    try:
        server = A3CPolicyServer(pol, q, pool)
        ready = []
        while len(ready) < pool.num_workers:
            ready, _ = pool.wait_ready(120)
        server.serve([0, 1])
        pool.reply(ready)
        pool.close()
        assert not server._s.value
        with pytest.raises(ValueError, match="closed"):
            server.serve([0])
        server.close()
    finally:
        pool.close()
        pol.close()
        q.close()
    assert _no_children()
