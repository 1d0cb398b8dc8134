"""The IMPALA policy server on the GPU (drl_policy_server_*, actor_server.py): the engine's batch-composition
invariance it rests on, the trajectories it commits against a serial n = 1 oracle that follows VectorActor's rules,
the queue's backpressure on the workers, an end-to-end run beside a training learner, and its argument checks."""
import ctypes as C
import functools
import mmap
import multiprocessing as mp
import threading
import time

import numpy as np
import pytest

T, A, L = 20, 18, 256
SHAPE = (84, 84, 4)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def N(native):
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
        if self.rng.rand() < 0.15:
            self.lives -= 1
        done = self.lives == 0 or self.t >= 25 + (a % 7)
        return self._frame(), float(self.rng.randint(0, 3)), done, {"ale.lives": self.lives}


def _params(seed=7, num_action=A):
    from distributed_reinforcement_learning_b200.model import impala_actor_critic
    p = impala_actor_critic.init_params(seed=seed, num_action=num_action, lstm_hidden_size=L, input_shape=SHAPE)
    rng = np.random.default_rng(seed + 1)
    return (p + rng.standard_normal(p.shape).astype(np.float32) * 0.01).astype(np.float32)


def _policy(params, max_batch=64, graph=True):
    from distributed_reinforcement_learning_b200.policy import NativePolicy
    p = NativePolicy(max_batch, num_action=A, use_cuda_graph=graph)
    p.set_params(params)
    return p


def _queue(queue_size, batch, trajectory=T, num_action=A):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import DeviceFIFOQueue
    return DeviceFIFOQueue(trajectory, SHAPE, num_action, queue_size, batch, 1, L)


def _pool(num_envs, per_worker, seed0=100):
    from distributed_reinforcement_learning_b200.actor_server import EnvWorkerPool
    return EnvWorkerPool([functools.partial(SynthEnv, seed0 + i) for i in range(num_envs)], [A] * num_envs,
                         per_worker, seeds=[seed0 + 1000 + i for i in range(num_envs)])


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
    """A row's policy, h, c and action do not depend on the other rows of its batch or on its position: the server
    serves any subset of environments in any order, and its bit-equality with the n = 1 oracle rests on this."""
    pol = _policy(_params())
    try:
        rng = np.random.RandomState(3)
        n = 64
        st = rng.randint(0, 256, (n,) + SHAPE).astype(np.uint8)
        pa = rng.randint(0, A, n).astype(np.int32)
        h = rng.standard_normal((n, L)).astype(np.float32) * 0.5
        c = rng.standard_normal((n, L)).astype(np.float32) * 0.5
        u = rng.random_sample(n)
        full = pol.act(st, pa, h, c, uniform=u)

        def same(out, i, r):
            for k in ("policy", "h", "c", "action"):
                assert np.array_equal(out[k][i], full[k][r]), (k, i, r)

        for r in (0, 63, 17):
            same(pol.act(st[r:r + 1], pa[r:r + 1], h[r:r + 1], c[r:r + 1], uniform=u[r:r + 1]), 0, r)
        # row 5 at row 0 and at row 63 of a batch of 64 others, and among random rows of batches of 1..64
        for pos in (0, 63):
            idx = np.array([i for i in range(n) if i != 5][:63])
            idx = np.insert(idx, pos, 5)
            out = pol.act(st[idx], pa[idx], h[idx], c[idx], uniform=u[idx])
            for i, r in enumerate(idx):
                same(out, i, r)
        for m in (2, 9, 33, 64):
            idx = rng.permutation(n)[:m]
            out = pol.act(st[idx], pa[idx], h[idx], c[idx], uniform=u[idx])
            for i, r in enumerate(idx):
                same(out, i, r)
    finally:
        pol.close()


def _oracle(pol, seed0, num_envs, unrolls):
    """Per task: its own env and RandomState, NativePolicy.act at n = 1 with host h and c, VectorActor's rules.
    -> the trajectories of `unrolls` unrolls of every task, as the queue stores them."""
    from distributed_reinforcement_learning_b200 import utils
    from distributed_reinforcement_learning_b200.actor_server import _Stats
    out = []
    for i in range(num_envs):
        env, rs = SynthEnv(seed0 + i), np.random.RandomState(seed0 + 1000 + i)
        stats = _Stats(1)
        state, pa = env.reset(), 0
        h, c = np.zeros((1, L), np.float32), np.zeros((1, L), np.float32)
        for _ in range(unrolls):
            tr = {k: [] for k in ("state", "reward", "done", "behavior_policy", "action", "previous_action",
                                  "previous_h", "previous_c")}
            for _ in range(T):
                o = pol.act(state[None], np.array([pa], np.int32), h, c, uniform=np.array([rs.random_sample()]))
                a = int(o["action"][0])
                for k, v in (("state", state), ("behavior_policy", o["policy"][0]), ("action", a),
                             ("previous_action", pa), ("previous_h", h[0]), ("previous_c", c[0])):
                    tr[k].append(v)
                _, r, d, state, ep = utils.impala_env_step(env, a, A, stats, 0, o["max_prob"][0])
                tr["reward"].append(r)
                tr["done"].append(d)
                if ep is None:
                    pa, h, c = a, o["h"].copy(), o["c"].copy()
                else:
                    pa, h, c = 0, np.zeros((1, L), np.float32), np.zeros((1, L), np.float32)
            out.append(dict(state=np.stack(tr["state"]), reward=np.array(tr["reward"], np.float32),
                            done=np.array(tr["done"], np.bool_), behavior_policy=np.stack(tr["behavior_policy"]),
                            action=np.array(tr["action"], np.int32),
                            previous_action=np.array(tr["previous_action"], np.int32),
                            previous_h=np.stack(tr["previous_h"]), previous_c=np.stack(tr["previous_c"])))
    return out


@pytest.mark.parametrize("graph", [True, False], ids=["graph", "eager"])
def test_served_trajectories_match_serial_oracle(N, graph):
    from distributed_reinforcement_learning_b200.actor_server import PolicyServer
    P, k, U = 3, 4, 3
    E = P * k
    params = _params(11)
    pol = _policy(params, max_batch=8, graph=graph)
    q = _queue(E * U, E)
    pool = _pool(E, k)
    server = None
    try:
        server = PolicyServer(pol, q, pool)
        # U unrolls and the reports carrying the last one's final rewards
        _serve_lockstep(server, pool, U * T + 1, np.random.RandomState(5), 8)
        assert q.get_size() == E * U
        got = [q.read(j) for j in range(E * U)]
    finally:
        if server is not None:
            server.close()
        pool.close()
    oracle_pol = _policy(params, max_batch=1, graph=graph)
    try:
        want = _oracle(oracle_pol, 100, E, U)
    finally:
        oracle_pol.close()
    q.close()
    pol.close()
    by_frames = {w["state"].tobytes(): w for w in want}
    assert len(by_frames) == len(want)
    matched = set()
    for g in got:
        key = g["state"].tobytes()
        assert key in by_frames and key not in matched
        matched.add(key)
        w = by_frames[key]
        for f in w:
            assert g[f].dtype == w[f].dtype and np.array_equal(g[f].view(np.uint8), w[f].view(np.uint8)), f
    assert len(matched) == len(want)
    assert _no_children()


def test_full_queue_blocks_serve_until_the_learner_pops(N):
    from distributed_reinforcement_learning_b200.actor_server import PolicyServer
    from distributed_reinforcement_learning_b200.agent import impala
    Ts, E = 5, 4
    q = _queue(E, E, trajectory=Ts)          # two slots of 4: two unrolls fit
    ag = impala.Agent(trajectory=Ts, input_shape=SHAPE, num_action=A, lstm_hidden_size=L, discount_factor=0.99,
                      start_learning_rate=6e-4, end_learning_rate=0.0, learning_frame=1e9, baseline_loss_coef=0.5,
                      entropy_coef=0.01, gradient_clip_norm=40.0, reward_clipping="abs_one",
                      model_name="server_bp", learner_name="server_bp")
    pol = _policy(_params(2), max_batch=4)
    pool = _pool(E, 2, seed0=300)
    server = None
    try:
        server = PolicyServer(pol, q, pool)
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
        losses = ag.train_from_queue(q)
        assert np.isfinite(losses).all() and q.get_size() == E
        server.serve(ids, timeout_ms=10000)
        pool.reply(ready)
        assert q.get_size() == 2 * E and (pool.views["action"][:E] >= 0).all()
        for _ in range(2):
            ag.train_from_queue(q)
        assert q.get_size() == 0   # 3 unrolls of 4 environments committed, 3 batches of 4 popped
    finally:
        if server is not None:
            server.close()
        pool.close()
        pol.close()
        q.close()
    assert _no_children()


def test_end_to_end_with_training_learner(N):
    from distributed_reinforcement_learning_b200.actor_server import PolicyServer
    from distributed_reinforcement_learning_b200.agent import impala
    B, steps = 8, 6
    ag = impala.Agent(trajectory=T, input_shape=SHAPE, num_action=A, lstm_hidden_size=L, discount_factor=0.99,
                      start_learning_rate=6e-4, end_learning_rate=0.0, learning_frame=1e9, baseline_loss_coef=0.5,
                      entropy_coef=0.01, gradient_clip_norm=40.0, reward_clipping="abs_one",
                      model_name="server_e2e", learner_name="server_e2e")
    ag._ensure_init()
    ag._params = _params(4)
    ag._get_engine(B)
    before = ag._engine.get_params()
    q = _queue(32, B)
    pol = _policy(_params(9))
    pool = _pool(24, 2, seed0=500)
    assert pool.num_workers == 12
    server = PolicyServer(pol, q, pool, learner=ag)
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
    assert all(set(e) == {"task", "episode", "score", "episode_step", "prob"} for e in episodes)
    pol.close()
    q.close()
    assert _no_children()


class _Block:
    """An exchange block without workers: page-aligned anonymous memory."""

    def __init__(self, num_envs, size=None, offset=0):
        from distributed_reinforcement_learning_b200.actor_server import exchange_bytes
        self.num_envs = num_envs
        self.exchange_bytes = exchange_bytes(num_envs) if size is None else size
        self._m = mmap.mmap(-1, exchange_bytes(num_envs) + mmap.PAGESIZE)
        self._anchor = C.c_char.from_buffer(self._m)
        self.address = C.addressof(self._anchor) + offset


def _create(N, pol, q, blk):
    s = C.c_void_p()
    rc = N.lib.drl_policy_server_create(pol._h, q._q, blk.num_envs, C.c_void_p(blk.address), blk.exchange_bytes,
                                        C.byref(s))
    return rc, s


def test_argument_checks_and_reregistration(N):
    from distributed_reinforcement_learning_b200.actor_server import PolicyServer
    pol = _policy(_params(1), max_batch=4)
    q = _queue(8, 4)
    blk = _Block(6)
    try:
        for bad in (_Block(6, offset=16), _Block(6, size=_Block(6).exchange_bytes - 1)):
            rc, _ = _create(N, pol, q, bad)
            assert rc == N.DRL_ERR_INVALID
        rc, _ = _create(N, pol, q, _Block(257, size=1 << 24))
        assert rc == N.DRL_ERR_INVALID
        for other in (_queue(8, 4, num_action=A + 1),):
            with pytest.raises(N.DrlError, match="num_action"):
                PolicyServer(pol, other, blk)
            other.close()
        server = PolicyServer(pol, q, blk)
        for ids in ([6], [-1], [0, 2, 0], [0, 1, 2, 3, 4]):
            with pytest.raises(N.DrlError) as e:
                server.serve(ids)
            assert e.value.code == N.DRL_ERR_INVALID
        server.close()
        # the block was unregistered: it can be registered again
        server = PolicyServer(pol, q, blk)
        server.close()
    finally:
        pol.close()
        q.close()


def test_closing_the_pool_closes_its_server(N):
    """The pool frees the exchange block only after its server has unregistered it."""
    from distributed_reinforcement_learning_b200.actor_server import PolicyServer
    pol = _policy(_params(1), max_batch=4)
    q = _queue(8, 4)
    pool = _pool(2, 1, seed0=700)
    try:
        server = PolicyServer(pol, q, pool)
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
