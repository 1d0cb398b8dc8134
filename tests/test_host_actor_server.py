"""The host side of the IMPALA policy server (actor_server.py), without a GPU: the exchange block's layout against
include/drl_b200.h, the shared environment step rule against VectorActor, and the worker pool's processes (spawned,
torch-free, failures surfaced by task, nothing left behind).  The replies the server's kernels would write are written
by the test itself."""
import functools
import multiprocessing as mp
import os
import re
import time

import numpy as np
import pytest

from distributed_reinforcement_learning_b200 import actor_server as S
from distributed_reinforcement_learning_b200 import utils

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class ScriptedEnv:
    """Frames that encode (seed, step), a life lost every `life_every` steps and an episode end every `episode_len`
    steps; step `fail_at` raises."""

    def __init__(self, seed, life_every=3, episode_len=7, fail_at=None):
        self.seed, self.life_every, self.episode_len, self.fail_at = seed, life_every, episode_len, fail_at
        self.calls = 0

    def _frame(self):
        f = np.zeros(S.FRAME_SHAPE, np.uint8)
        f[0, 0, 0], f[0, 0, 1] = self.seed, self.calls % 256
        return f

    def reset(self):
        self.t, self.lives = 0, 5
        return self._frame()

    def step(self, a):
        self.calls += 1
        if self.fail_at is not None and self.calls >= self.fail_at:
            raise ValueError("scripted failure of env %d" % self.seed)
        self.t += 1
        if self.t % self.life_every == 0:
            self.lives -= 1
        return self._frame(), float(a % 3), self.t >= self.episode_len, {"ale.lives": self.lives}


def _no_children():
    deadline = time.time() + 10
    while mp.active_children() and time.time() < deadline:
        time.sleep(0.05)
    return not mp.active_children()


def test_exchange_layout_matches_header():
    with open(os.path.join(ROOT, "include", "drl_b200.h")) as f:
        defs = {k: int(v) for k, v in re.findall(r"#define DRL_SERVER_(\w+) (\d+)", f.read())}
    assert defs == dict(REPORT_FRAME=S.REPORT_FRAME, REPORT_UNIFORM=S.REPORT_UNIFORM, REPORT_REWARD=S.REPORT_REWARD,
                        REPORT_DONE=S.REPORT_DONE, REPORT_RESET=S.REPORT_RESET, REPORT_BYTES=S.REPORT_BYTES,
                        REPLY_ACTION=S.REPLY_ACTION, REPLY_MAX_PROB=S.REPLY_MAX_PROB, REPLY_BYTES=S.REPLY_BYTES)
    frame = int(np.prod(S.FRAME_SHAPE))
    # every field 16-byte aligned, in order, no overlap
    offs = [S.REPORT_FRAME, S.REPORT_UNIFORM, S.REPORT_REWARD, S.REPORT_DONE, S.REPORT_RESET]
    ends = [frame, S.REPORT_UNIFORM + 8, S.REPORT_REWARD + 4, S.REPORT_DONE + 1, S.REPORT_RESET + 1]
    assert all(o % 16 == 0 for o in offs + [S.REPORT_BYTES, S.REPLY_ACTION, S.REPLY_MAX_PROB, S.REPLY_BYTES])
    assert all(ends[i] <= offs[i + 1] for i in range(len(offs) - 1)) and ends[-1] <= S.REPORT_BYTES
    assert S.REPLY_ACTION + 4 <= S.REPLY_MAX_PROB and S.REPLY_MAX_PROB + 4 <= S.REPLY_BYTES
    for n in (1, 3, 12, 64, 256):
        b = S.exchange_bytes(n)
        assert b % S.PAGE == 0 and n * (S.REPORT_BYTES + S.REPLY_BYTES) <= b < n * (S.REPORT_BYTES + S.REPLY_BYTES) + S.PAGE


def test_exchange_views_address_the_records():
    n = 5
    buf = bytearray(S.exchange_bytes(n))
    v = S.exchange_views(buf, n)
    v["frame"][3] = 7
    v["uniform"][3] = 0.25
    v["reward"][3], v["done"][3], v["reset"][3] = -1.0, 1, 1
    v["action"][2], v["max_prob"][2] = 11, 0.5
    raw = np.frombuffer(buf, np.uint8)
    r3 = 3 * S.REPORT_BYTES
    assert (raw[r3:r3 + 28224] == 7).all() and raw[r3 + 28224:r3 + S.REPORT_BYTES].any()
    assert np.frombuffer(buf, np.float64, 1, r3 + S.REPORT_UNIFORM)[0] == 0.25
    assert np.frombuffer(buf, np.float32, 1, r3 + S.REPORT_REWARD)[0] == -1.0
    assert raw[r3 + S.REPORT_DONE] == 1 and raw[r3 + S.REPORT_RESET] == 1
    rp = n * S.REPORT_BYTES + 2 * S.REPLY_BYTES
    assert np.frombuffer(buf, np.int32, 1, rp + S.REPLY_ACTION)[0] == 11
    assert np.frombuffer(buf, np.float32, 1, rp + S.REPLY_MAX_PROB)[0] == 0.5
    # nothing else was written
    assert raw[:r3].sum() == 0 and raw[r3 + S.REPORT_BYTES:n * S.REPORT_BYTES].sum() == 0


class _FakePolicy:
    """NativePolicy.act's interface with a scripted rule: action = (frame[0,0,1] + previous action) % A."""
    max_batch, L, A = 64, 4, 6

    def act(self, state, previous_action, h, c):
        n = len(state)
        action = ((state[:, 0, 0, 1].astype(np.int64) + previous_action) % self.A).astype(np.int32)
        policy = np.full((n, self.A), 0.1, np.float32)
        policy[np.arange(n), action] = 0.5
        return dict(action=action, policy=policy, max_prob=policy.max(-1), h=h + 1, c=c - 1)


class _ListQueue:
    def __init__(self):
        self.items = []

    def append_to_queue(self, task, **kw):
        self.items.append((task, kw))


def _expected_records(actions, avail, life_every, episode_len, task):
    """What the IMPALA actor's rules give for ScriptedEnv under the recorded actions, derived without the step rule:
    per step (reward, done, previous action, steps since the episode started), and the finished episodes."""
    rows, episodes = [], []
    t, episode, score, pa = 0, 0, 0.0, 0
    for a in actions:
        t += 1
        raw = float((a % avail) % 3)
        lost = t % life_every == 0
        rows.append((-1.0 if lost else raw, lost, pa, t - 1))
        score += raw
        pa = a
        if t >= episode_len:
            episodes.append(dict(task=task, episode=episode, score=score, episode_step=t, prob=0.5))
            t, episode, score, pa = 0, episode + 1, 0.0, 0
    return rows, episodes


def test_step_rule_gives_vector_actor_records():
    """VectorActor (through utils.impala_env_step) against expectations worked out from the environments' script:
    lost lives as reward -1 and done, the raw reward of `action % available_action`, the unmodified action, and the
    previous action, h and c back to 0 at every episode start."""
    from distributed_reinforcement_learning_b200.actor import VectorActor
    n, T = 3, 5
    avail = [4, 6, 5]
    q = _ListQueue()
    actor = VectorActor(_FakePolicy(), [ScriptedEnv(i, 3 + i, 7 + i) for i in range(n)], q, T, avail)
    episodes = [ep for _ in range(4) for ep in actor.run_unroll()]
    got = {i: [] for i in range(n)}
    for task, kw in q.items:
        got[task] += [(int(a), float(r), bool(d), int(pa), h, c) for a, r, d, pa, h, c in zip(
            kw["unrolled_action"], kw["unrolled_reward"], kw["unrolled_done"], kw["unrolled_previous_action"],
            kw["unrolled_previous_h"], kw["unrolled_previous_c"])]
    want_episodes = []
    for i in range(n):
        assert len(got[i]) == 4 * T
        actions = [r[0] for r in got[i]]
        rows, eps = _expected_records(actions, avail[i], 3 + i, 7 + i, i)
        want_episodes += eps
        for (a, r, d, pa, h, c), (wr, wd, wpa, since) in zip(got[i], rows):
            assert (r, d, pa) == (wr, wd, wpa)
            # _FakePolicy adds 1 to h and subtracts 1 from c per act: both count the acts since the episode began
            assert (h == since).all() and (c == -since).all()
    key = lambda e: (e["task"], e["episode"])
    assert sorted(episodes, key=key) == sorted(want_episodes, key=key) and len(episodes) >= n


def _serve_on_cpu(pool, rounds, action=1):
    """Drives the pool as the server would, writing every reply itself: `rounds` steps of every environment."""
    episodes = []
    for _ in range(rounds):
        ready = []
        while len(ready) < pool.num_workers:
            ready, eps = pool.wait_ready(60)
            episodes += eps
        for w in ready:
            for e in pool.env_ids(w):
                pool.views["action"][e], pool.views["max_prob"][e] = action, 0.5
        pool.reply(ready)
    return episodes


def test_pool_spawns_torch_free_workers_and_closes():
    import torch  # noqa: F401  (imported here, so a worker that inherited the parent's modules would show it)
    fns = [functools.partial(ScriptedEnv, i) for i in range(5)]
    with S.EnvWorkerPool(fns, [4] * 5, 2, seeds=range(5)) as pool:
        assert pool.num_workers == 3 and [pool.env_ids(w) for w in range(3)] == [[0, 1], [2, 3], [4]]
        assert len(pool.worker_info) == 3
        assert not any(i["torch"] or i["native"] for i in pool.worker_info)
        assert all(type(x["process"]).__name__ == "SpawnProcess" for x in pool._workers)
        v = pool.views
        assert (v["reset"][:5] == 1).all()
        u0 = v["uniform"][:5].copy()
        assert np.array_equal(u0, [np.random.RandomState(i).random_sample() for i in range(5)])
        episodes = _serve_on_cpu(pool, 12)
        while len(pool.wait_ready(60)[0]) < 3:
            pass
        # each environment's draws come from its own stream, whatever the grouping
        assert np.array_equal(v["uniform"][:5], [np.random.RandomState(i).random_sample(13)[-1] for i in range(5)])
        # action 1 throughout: raw reward 1 per step, one 7-step episode each, then steps 1..5 of the next one
        key = lambda e: e["task"]
        assert sorted(episodes, key=key) == [dict(task=i, episode=0, score=7.0, episode_step=7, prob=0.5)
                                             for i in range(5)]
        assert (v["reward"][:5] == 1.0).all() and (v["done"][:5] == 0).all() and (v["reset"][:5] == 0).all()
        assert (v["frame"][:5, 0, 0, 1] == 12).all() and (v["frame"][:5, 0, 0, 0] == np.arange(5)).all()
    assert _no_children()


def test_closing_the_pool_closes_its_servers_first():
    fns = [functools.partial(ScriptedEnv, i) for i in range(2)]
    pool = S.EnvWorkerPool(fns, [4] * 2, 1, seeds=range(2))
    order = []

    class Server:   # what PolicyServer does with its pool
        def close(self):
            order.append(("server", pool._shm is not None))
            pool._unbind(self)

    srv = Server()
    pool._bind(srv)
    pool.close()
    assert order == [("server", True)] and pool._servers == []
    with pytest.raises(ValueError):
        pool._bind(srv)
    assert _no_children()


def test_worker_failure_names_the_task_and_leaves_no_children():
    fns = [functools.partial(ScriptedEnv, i) for i in range(4)]
    fns[2] = functools.partial(ScriptedEnv, 2, fail_at=3)
    pool = S.EnvWorkerPool(fns, [4] * 4, 2, seeds=range(4))
    try:
        with pytest.raises(RuntimeError, match="environment task 2 raised"):
            _serve_on_cpu(pool, 10)
    finally:
        pool.close()
    assert _no_children()


def test_env_factory_that_raises_at_start_is_reported():
    fns = [functools.partial(ScriptedEnv, 0), functools.partial(ScriptedEnv, "not a seed")]
    with pytest.raises(RuntimeError, match="environment task 1 raised"):
        S.EnvWorkerPool(fns, [4, 4], 1, seeds=[0, 1])
    assert _no_children()


def test_unpicklable_env_factory_is_rejected():
    with pytest.raises(ValueError, match=r"env_fns\[1\] cannot be pickled"):
        S.EnvWorkerPool([functools.partial(ScriptedEnv, 0), lambda: ScriptedEnv(1)], [4, 4], 1, seeds=[0, 1])
    assert _no_children()


def test_pool_argument_checks():
    fn = functools.partial(ScriptedEnv, 0)
    with pytest.raises(ValueError):
        S.EnvWorkerPool([fn] * 2, [4], 1, seeds=[0, 1])
    with pytest.raises(ValueError):
        S.EnvWorkerPool([fn] * 257, [4] * 257, 1, seeds=range(257))
    with pytest.raises(ValueError):
        S.EnvWorkerPool([fn], [4], 0, seeds=[0])
