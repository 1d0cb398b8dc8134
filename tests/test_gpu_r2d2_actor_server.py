"""The R2D2 policy server on the GPU (drl_r2d2_policy_server_*, actor_server.py: R2D2PolicyServer): the R2D2 engine's
batch-composition invariance it rests on, the sequences it commits against a serial n = 1 oracle that follows
R2D2VectorActor's rules, the queue's backpressure on the workers, an end-to-end run beside a training learner, a
malformed explore value in the exchange block, and its argument checks."""
import ctypes as C
import functools
import mmap
import multiprocessing as mp
import threading
import time

import numpy as np
import pytest

S, BURN_IN, A, L = 15, 7, 4, 64

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def N(native):
    if native.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return native


class SynthEnv:
    """A cheap seeded stand-in for an Atari environment: random 84x84xC frames, rewards in {0, 1, 2}, a life lost now
    and then and short episodes, so that sequences cross life losses and episode ends."""

    def __init__(self, seed, channels=1):
        self.rng = np.random.RandomState(seed)
        self.shape = (84, 84, channels)

    def _frame(self):
        return self.rng.randint(0, 256, self.shape).astype(np.uint8)

    def reset(self):
        self.lives, self.t = 5, 0
        return self._frame()

    def step(self, a):
        self.t += 1
        if self.rng.rand() < 0.1:
            self.lives -= 1
        done = self.lives == 0 or self.t >= 18 + (a % 5)
        return self._frame(), float(self.rng.randint(0, 3)), done, {"ale.lives": self.lives}


def _params(seed=3, channels=1):
    from distributed_reinforcement_learning_b200.model import r2d2_lstm
    p = r2d2_lstm.init_params(seed, num_action=A, lstm_size=L, input_shape=(84, 84, channels))
    rng = np.random.default_rng(seed + 1)
    return (p + rng.standard_normal(p.shape).astype(np.float32) * 0.01).astype(np.float32)


def _policy(params, max_batch=64, graph=True, channels=1):
    from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
    p = NativeR2D2Policy(max_batch, num_action=A, lstm_size=L, input_shape=(84, 84, channels), use_cuda_graph=graph)
    p.set_params(params)
    return p


def _queue(queue_size, batch, channels=1, num_action=A):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import R2D2DeviceFIFOQueue
    return R2D2DeviceFIFOQueue(S, (84, 84, channels), num_action, queue_size, batch, 1, L)


def _pool(num_envs, per_worker, seed0=100, channels=1):
    from distributed_reinforcement_learning_b200.actor_server import R2D2EnvWorkerPool
    return R2D2EnvWorkerPool([functools.partial(SynthEnv, seed0 + i, channels) for i in range(num_envs)], A,
                             per_worker, seeds=[seed0 + 1000 + i for i in range(num_envs)], channels=channels)


def _agent(name, params, graph=True):
    from distributed_reinforcement_learning_b200.agent import r2d2
    from distributed_reinforcement_learning_b200.model import r2d2_lstm
    a = r2d2.Agent(S, BURN_IN, [84, 84, 1], A, L, 0.997, 1e-4, 1e-4, 1e9, 40.0, name, name)
    a.use_cuda_graph = graph
    a._main = params.copy()
    a._target = r2d2_lstm.init_params(11, num_action=A, lstm_size=L, input_shape=(84, 84, 1))
    z = np.zeros_like(a._main)
    a._opt = dict(m=z, v=z.copy(), step=0, beta1_power=0.9, beta2_power=0.999)
    return a


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
    """A row's q, h, c, action and q_action do not depend on the other rows of its batch or on its position, greedy
    rows and explore rows alike: the server serves any subset of environments in any order, and its bit-equality with
    the n = 1 oracle rests on this."""
    pol = _policy(_params())
    try:
        rng = np.random.RandomState(3)
        n = 64
        st = rng.randint(0, 256, (n, 84, 84, 1)).astype(np.uint8)
        pa = rng.randint(0, A, n).astype(np.int32)
        h = rng.standard_normal((n, L)).astype(np.float32) * 0.5
        c = rng.standard_normal((n, L)).astype(np.float32) * 0.5
        ex = np.where(rng.rand(n) < 0.5, -1, rng.randint(0, A, n)).astype(np.int32)
        assert (ex == -1).any() and (ex >= 0).any()
        full = pol.act(st, pa, h, c, explore_action=ex)

        def same(out, i, r):
            for k in ("q", "h", "c", "action", "q_action"):
                assert np.array_equal(out[k][i], full[k][r]), (k, i, r)

        for r in (0, 63, 17):
            same(pol.act(st[r:r + 1], pa[r:r + 1], h[r:r + 1], c[r:r + 1], explore_action=ex[r:r + 1]), 0, r)
        for pos in (0, 63):
            idx = np.insert(np.array([i for i in range(n) if i != 5][:63]), pos, 5)
            out = pol.act(st[idx], pa[idx], h[idx], c[idx], explore_action=ex[idx])
            for i, r in enumerate(idx):
                same(out, i, r)
        for m in range(1, 65):
            idx = rng.permutation(n)[:m]
            out = pol.act(st[idx], pa[idx], h[idx], c[idx], explore_action=ex[idx])
            for i, r in enumerate(idx):
                same(out, i, r)
    finally:
        pol.close()


def _oracle(pol, seed0, num_envs, unrolls, channels=1):
    """Per task: its own env and RandomState, NativeR2D2Policy.act at n = 1 with host h and c, R2D2VectorActor's rules
    (utils.r2d2_env_step).  -> the sequences of `unrolls` unrolls of every task, as the queue stores them."""
    from distributed_reinforcement_learning_b200 import utils
    from distributed_reinforcement_learning_b200.actor_server import _R2D2Stats, explore_action
    out = []
    for i in range(num_envs):
        env, rs = SynthEnv(seed0 + i, channels), np.random.RandomState(seed0 + 1000 + i)
        stats = _R2D2Stats(1)
        state, pa = env.reset(), 0
        h, c = np.zeros((1, L), np.float32), np.zeros((1, L), np.float32)
        for _ in range(unrolls):
            rec = {k: [] for k in ("state", "previous_action", "action", "reward", "done")}
            h0, c0 = h[0].copy(), c[0].copy()
            for _ in range(S):
                ex = explore_action(rs, stats.epsilon[0], A)
                o = pol.act(state[None], np.array([pa], np.int32), h, c, explore_action=np.array([ex], np.int32))
                a = int(o["action"][0])
                for k, v in (("state", state), ("previous_action", pa), ("action", a)):
                    rec[k].append(v)
                _, r, d, state, ep = utils.r2d2_env_step(env, a, stats, 0, o["q_action"][0])
                rec["reward"].append(r)
                rec["done"].append(d)
                if ep is None:
                    pa, h, c = a, o["h"].copy(), o["c"].copy()
                else:
                    pa, h, c = 0, np.zeros((1, L), np.float32), np.zeros((1, L), np.float32)
            out.append(dict(state=np.stack(rec["state"]), previous_action=np.array(rec["previous_action"], np.int32),
                            action=np.array(rec["action"], np.int32), reward=np.array(rec["reward"], np.float32),
                            done=np.array(rec["done"], np.bool_), previous_h=h0, previous_c=c0))
    return out


def _check_against_oracle(got, want):
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


@pytest.mark.parametrize("graph,channels", [(True, 1), (False, 1), (True, 4)], ids=["graph", "eager", "graph-c4"])
def test_served_sequences_match_serial_oracle(N, graph, channels):
    from distributed_reinforcement_learning_b200.actor_server import R2D2PolicyServer
    P, k, U = 3, 4, 3
    E = P * k
    params = _params(11, channels)
    pol = _policy(params, max_batch=8, graph=graph, channels=channels)
    q = _queue(E * U, E, channels)
    pool = _pool(E, k, channels=channels)
    server = None
    try:
        server = R2D2PolicyServer(pol, q, pool)
        # U sequences and the reports carrying the last one's final rewards
        _serve_lockstep(server, pool, U * S + 1, np.random.RandomState(5), 8)
        assert q.get_size() == E * U
        got = [q.read(j) for j in range(E * U)]
    finally:
        if server is not None:
            server.close()
        pool.close()
    oracle_pol = _policy(params, max_batch=1, graph=graph, channels=channels)
    try:
        want = _oracle(oracle_pol, 100, E, U, channels)
    finally:
        oracle_pol.close()
    q.close()
    pol.close()
    assert any(w["done"].any() for w in want) and any((w["previous_action"] == 0).sum() > 1 for w in want)
    _check_against_oracle(got, want)
    assert _no_children()


def test_full_queue_blocks_serve_until_the_learner_pops(N):
    from distributed_reinforcement_learning_b200.actor_server import R2D2PolicyServer
    E = 4
    q = _queue(E, E)          # two slots of 4: two sequences per environment fit
    ag = _agent("r2d2_server_bp", _params(2))
    memory = ag.device_memory(64)
    pol = _policy(_params(2), max_batch=4)
    pool = _pool(E, 2, seed0=300)
    server = None
    try:
        server = R2D2PolicyServer(pol, q, pool)
        rng = np.random.RandomState(1)
        _serve_lockstep(server, pool, 2 * S + 1, rng, 4)
        assert q.get_size() == 2 * E
        _serve_lockstep(server, pool, S - 1, rng, 4)      # the third sequence up to its last step
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
        memory.add_from_queue(q)
        assert q.get_size() == E and memory.n_entries == E
        server.serve(ids, timeout_ms=10000)
        pool.reply(ready)
        assert q.get_size() == 2 * E and (pool.views["action"][:E] >= 0).all()
        for _ in range(2):
            memory.add_from_queue(q)
        assert q.get_size() == 0 and memory.n_entries == 3 * E
        loss, td = ag.train_from_memory(memory, E)
        assert np.isfinite(loss) and np.isfinite(td).all()
    finally:
        if server is not None:
            server.close()
        pool.close()
        pol.close()
        memory.close()
        q.close()
    assert _no_children()


def test_end_to_end_with_training_learner(N):
    from distributed_reinforcement_learning_b200.actor_server import R2D2PolicyServer
    B, steps = 8, 6
    ag = _agent("r2d2_server_e2e", _params(4))
    memory = ag.device_memory(256)
    q = _queue(32, B)
    pol = _policy(_params(9))
    pool = _pool(16, 2, seed0=500)
    assert pool.num_workers == 8
    server = R2D2PolicyServer(pol, q, pool, learner=ag)
    stop, losses, errors, episodes = threading.Event(), [], [], []

    def serve():
        try:
            server.run(stop, on_episodes=episodes.extend)
        except Exception as e:   # pragma: no cover - reported below
            errors.append(e)

    th = threading.Thread(target=serve)
    th.start()
    try:
        memory.add_from_queue(q, timeout_ms=120000)
        before = ag._engine.get_params()
        for _ in range(steps):
            memory.add_from_queue(q, timeout_ms=120000)
            losses.append(ag.train_from_memory(memory, B)[0])
    finally:
        stop.set()
        th.join(60)
        server.close()
        pool.close()
    assert not th.is_alive() and not errors
    assert np.isfinite(np.array(losses)).all() and ag.train_calls == steps
    assert not np.array_equal(ag._engine.get_params(), before)
    assert server.syncs >= 2 and sum(server.batch_sizes.values()) > 0
    assert all(set(e) == {"task", "episode", "score", "epsilon", "episode_step", "avg_q_value"} for e in episodes)
    memory.close()
    pol.close()
    q.close()
    assert _no_children()


class _Block:
    """An exchange block without workers: page-aligned anonymous memory, with the R2D2 views of its records."""

    def __init__(self, num_envs, size=None, offset=0, channels=1):
        from distributed_reinforcement_learning_b200.actor_server import exchange_bytes, r2d2_exchange_views
        self.num_envs = num_envs
        self.exchange_bytes = exchange_bytes(num_envs) if size is None else size
        self._m = mmap.mmap(-1, exchange_bytes(num_envs) + mmap.PAGESIZE)
        self._anchor = C.c_char.from_buffer(self._m)
        self.address = C.addressof(self._anchor) + offset
        self.views = r2d2_exchange_views(self._m, num_envs, channels) if offset == 0 else None


def _create(N, pol, q, blk):
    s = C.c_void_p()
    rc = N.lib.drl_r2d2_policy_server_create(pol._h, q._q, blk.num_envs, C.c_void_p(blk.address), blk.exchange_bytes,
                                             C.byref(s))
    return rc, s


def test_malformed_explore_value_is_rejected_naming_the_environment(N):
    """An explore value outside [-1, A) written into the block by another process: DRL_ERR_INVALID naming the
    environment, before anything is reserved or launched, so the replies, the queue and the state table are as they
    were; once the value is fixed the environment is served at the step it was at."""
    from distributed_reinforcement_learning_b200.actor_server import R2D2PolicyServer
    params = _params(6)
    pol = _policy(params, max_batch=4)
    q = _queue(8, 4)
    blk = _Block(3)
    v = blk.views
    rng = np.random.RandomState(2)
    v["frame"][:] = rng.randint(0, 256, v["frame"].shape)
    v["explore"][:], v["reward"][:], v["done"][:], v["reset"][:] = -1, 0.0, 0, 1
    server = R2D2PolicyServer(pol, q, blk)
    ref = _policy(params, max_batch=1)
    try:
        server.serve([0, 1, 2])
        first = v["action"][:3].copy(), v["q_action"][:3].copy()
        v["reset"][:] = 0
        for bad in (A, -2, 1 << 30, -(1 << 31)):
            v["explore"][1] = bad
            v["action"][:3], v["q_action"][:3] = -7, -7.0
            with pytest.raises(N.DrlError, match="environment 1 reports explore action %d" % bad) as e:
                server.serve([0, 2, 1])
            assert e.value.code == N.DRL_ERR_INVALID
            assert (v["action"][:3] == -7).all() and (v["q_action"][:3] == -7.0).all() and q.get_size() == 0
        v["explore"][1] = 2
        server.serve([1])
        # environment 1's second act: its h and c from the first serve, the explore action 2
        o1 = ref.act(v["frame"][1:2], np.zeros(1, np.int32), np.zeros((1, L), np.float32),
                     np.zeros((1, L), np.float32), explore_action=np.array([-1], np.int32))
        assert o1["action"][0] == first[0][1] and o1["q_action"][0] == first[1][1]
        o2 = ref.act(v["frame"][1:2], o1["action"], o1["h"], o1["c"], explore_action=np.array([2], np.int32))
        assert v["action"][1] == 2 and v["q_action"][1] == o2["q_action"][0]
    finally:
        server.close()
        ref.close()
        pol.close()
        q.close()


def test_argument_checks_and_reregistration(N):
    from distributed_reinforcement_learning_b200.actor_server import R2D2PolicyServer
    pol = _policy(_params(1), max_batch=4)
    q = _queue(8, 4)
    blk = _Block(6)
    try:
        for bad in (_Block(6, offset=16), _Block(6, size=_Block(6).exchange_bytes - 1)):
            rc, _ = _create(N, pol, q, bad)
            assert rc == N.DRL_ERR_INVALID
        rc, _ = _create(N, pol, q, _Block(257, size=1 << 24))
        assert rc == N.DRL_ERR_INVALID
        for other, match in ((_queue(8, 4, num_action=A + 1), "num_action"), (_queue(8, 4, channels=4), "84x84x4"),
                             (_queue(2, 2), "sequences")):
            with pytest.raises(N.DrlError, match=match):
                R2D2PolicyServer(pol, other, blk)
            other.close()
        server = R2D2PolicyServer(pol, q, blk)
        for ids in ([6], [-1], [0, 2, 0], [0, 1, 2, 3, 4]):
            with pytest.raises(N.DrlError) as e:
                server.serve(ids)
            assert e.value.code == N.DRL_ERR_INVALID
        server.close()
        with pytest.raises(ValueError, match="closed"):
            server.serve([0])
        # the block was unregistered: it can be registered again
        server = R2D2PolicyServer(pol, q, blk)
        server.close()
    finally:
        pol.close()
        q.close()


def test_closing_the_pool_closes_its_server(N):
    """The pool frees the exchange block only after its server has unregistered it."""
    from distributed_reinforcement_learning_b200.actor_server import R2D2PolicyServer
    pol = _policy(_params(1), max_batch=4)
    q = _queue(8, 4)
    pool = _pool(2, 1, seed0=700)
    try:
        server = R2D2PolicyServer(pol, q, pool)
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
