"""The host side of the A3C policy server (actor_server.py: A3CEnvWorkerPool, A3CPolicyServer), without a GPU: the A3C
exchange records against include/drl_b200.h, the shared step rule utils.impala_env_step against A3CVectorActor's
records (next_state included), and the worker pool's processes (spawned, torch-free, next_state and reset written
after an episode end, failures surfaced by task, nothing left behind).  The replies the server's kernels would write
are written by the test itself."""
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
A = 4


class ScriptedEnv:
    """84x84x4 frames that encode (seed, step calls, resets), a life lost every `life_every` steps and an episode end
    every `episode_len` steps; step `fail_at` raises.  A reset frame differs from the episode's last frame."""

    def __init__(self, seed, life_every=3, episode_len=7, fail_at=None):
        self.seed, self.life_every, self.episode_len, self.fail_at = seed, life_every, episode_len, fail_at
        self.calls = self.resets = 0

    def _frame(self):
        f = np.zeros((84, 84, 4), np.uint8)
        f[0, 0, 0], f[0, 1, 0], f[0, 2, 0] = self.seed, self.calls % 256, self.resets % 256
        return f

    def reset(self):
        self.t, self.lives = 0, 5
        self.resets += 1
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


def test_a3c_exchange_layout_matches_header():
    with open(os.path.join(ROOT, "include", "drl_b200.h")) as f:
        defs = {k: int(v) for k, v in re.findall(r"#define DRL_A3C_SERVER_(\w+) (\d+)", f.read())}
    assert defs == dict(REPORT_FRAME=S.A3C_REPORT_FRAME, REPORT_NEXT_STATE=S.A3C_REPORT_NEXT_STATE,
                        REPORT_UNIFORM=S.A3C_REPORT_UNIFORM, REPORT_REWARD=S.A3C_REPORT_REWARD,
                        REPORT_DONE=S.A3C_REPORT_DONE, REPORT_RESET=S.A3C_REPORT_RESET,
                        REPORT_BYTES=S.A3C_REPORT_BYTES, REPLY_ACTION=S.A3C_REPLY_ACTION,
                        REPLY_MAX_PROB=S.A3C_REPLY_MAX_PROB, REPLY_BYTES=S.A3C_REPLY_BYTES)
    frame = 84 * 84 * 4
    offs = [S.A3C_REPORT_FRAME, S.A3C_REPORT_NEXT_STATE, S.A3C_REPORT_UNIFORM, S.A3C_REPORT_REWARD,
            S.A3C_REPORT_DONE, S.A3C_REPORT_RESET]
    ends = [frame, S.A3C_REPORT_NEXT_STATE + frame, S.A3C_REPORT_UNIFORM + 8, S.A3C_REPORT_REWARD + 4,
            S.A3C_REPORT_DONE + 1, S.A3C_REPORT_RESET + 1]
    assert all(o % 16 == 0 for o in offs + [S.A3C_REPORT_BYTES, S.A3C_REPLY_ACTION, S.A3C_REPLY_MAX_PROB,
                                            S.A3C_REPLY_BYTES])
    assert all(ends[i] <= offs[i + 1] for i in range(len(offs) - 1)) and ends[-1] <= S.A3C_REPORT_BYTES
    assert S.A3C_REPLY_ACTION + 4 <= S.A3C_REPLY_MAX_PROB and S.A3C_REPLY_MAX_PROB + 4 <= S.A3C_REPLY_BYTES
    # the replies have the other servers' size; the reports are larger, so the block is sized on its own
    assert S.A3C_REPLY_BYTES == S.REPLY_BYTES and S.A3C_REPORT_BYTES > S.REPORT_BYTES
    for n in (1, 3, 256):
        b = S.a3c_exchange_bytes(n)
        assert b % S.PAGE == 0 and n * (S.A3C_REPORT_BYTES + S.A3C_REPLY_BYTES) <= b < \
            n * (S.A3C_REPORT_BYTES + S.A3C_REPLY_BYTES) + S.PAGE
        assert b > S.exchange_bytes(n)


def test_a3c_exchange_views_address_the_records():
    n = 5
    buf = bytearray(S.a3c_exchange_bytes(n))
    v = S.a3c_exchange_views(buf, n)
    assert set(v) == {"frame", "next_state", "uniform", "reward", "done", "reset", "action", "max_prob"}
    assert v["frame"].shape == v["next_state"].shape == (n, 84, 84, 4)
    v["frame"][3] = 7
    v["next_state"][3] = 9
    v["uniform"][3] = 0.625
    v["reward"][3], v["done"][3], v["reset"][3] = -1.0, 1, 1
    v["action"][2], v["max_prob"][2] = 3, 0.5
    raw = np.frombuffer(buf, np.uint8)
    r3 = 3 * S.A3C_REPORT_BYTES
    frame = 84 * 84 * 4
    assert (raw[r3:r3 + frame] == 7).all()
    assert (raw[r3 + S.A3C_REPORT_NEXT_STATE:r3 + S.A3C_REPORT_NEXT_STATE + frame] == 9).all()
    assert np.frombuffer(buf, np.float64, 1, r3 + S.A3C_REPORT_UNIFORM)[0] == 0.625
    assert np.frombuffer(buf, np.float32, 1, r3 + S.A3C_REPORT_REWARD)[0] == -1.0
    assert raw[r3 + S.A3C_REPORT_DONE] == 1 and raw[r3 + S.A3C_REPORT_RESET] == 1
    rp = n * S.A3C_REPORT_BYTES + 2 * S.A3C_REPLY_BYTES
    assert np.frombuffer(buf, np.int32, 1, rp + S.A3C_REPLY_ACTION)[0] == 3
    assert np.frombuffer(buf, np.float32, 1, rp + S.A3C_REPLY_MAX_PROB)[0] == 0.5
    # nothing else was written
    rest = raw.copy()
    for off, size in ((S.A3C_REPORT_FRAME, 2 * frame), (S.A3C_REPORT_UNIFORM, 8), (S.A3C_REPORT_REWARD, 4),
                      (S.A3C_REPORT_DONE, 1), (S.A3C_REPORT_RESET, 1)):
        rest[r3 + off:r3 + off + size] = 0
    rest[rp:rp + S.A3C_REPLY_BYTES] = 0
    assert not rest.any()


class _FakeA3CPolicy:
    """NativeA3CPolicy.act's interface with a scripted rule: action = (frame[0,1,0] + 2 frame[0,2,0] + previous action)
    % A, max_prob = 0.125 (action + 1)."""
    max_batch, A = 64, A

    def act(self, state, previous_action):
        action = ((state[:, 0, 1, 0].astype(np.int64) + 2 * state[:, 0, 2, 0] + previous_action) % self.A)
        action = action.astype(np.int32)
        return dict(action=action, max_prob=(0.125 * (action + 1)).astype(np.float32))


class _ListQueue:
    def __init__(self):
        self.items = []

    def append_to_queue(self, task, **kw):
        self.items.append((task, kw))


def test_impala_step_rule_gives_a3c_vector_actor_records():
    """A3CVectorActor's host records against the same environments stepped under utils.impala_env_step with the
    actions the actor took: state, next_state (the terminal frame at an episode end, not the reset frame), reward -1
    and done on a life loss, the previous action back to 0 at an episode start, and the finished episodes."""
    from distributed_reinforcement_learning_b200.actor import A3CVectorActor
    n, T, unrolls = 3, 5, 5
    avail = [3, 4, 2]
    q = _ListQueue()
    actor = A3CVectorActor(_FakeA3CPolicy(), [ScriptedEnv(i, 3 + i, 7 + i) for i in range(n)], q, T, avail)
    episodes = [ep for _ in range(unrolls) for ep in actor.run_unroll()]
    got = {i: {k: [] for k in ("state", "next_state", "reward", "done", "action", "previous_action")}
           for i in range(n)}
    for task, kw in q.items:
        for k in got[task]:
            got[task][k].extend(list(kw["unrolled_" + k]))
    want_episodes = []
    for i in range(n):
        env = ScriptedEnv(i, 3 + i, 7 + i)
        stats = S._Stats(1)
        state, pa = env.reset(), 0
        g = got[i]
        assert len(g["action"]) == unrolls * T
        for k, a in enumerate(g["action"]):
            prob = np.float32(0.125 * (a + 1))
            next_state, r, d, new_state, ep = utils.impala_env_step(env, a, avail[i], stats, 0, prob, task=i)
            assert (g["state"][k] == state).all() and (g["next_state"][k] == next_state).all(), (i, k)
            assert (float(g["reward"][k]), bool(g["done"][k]), int(g["previous_action"][k])) == (r, d, pa), (i, k)
            if ep is not None:
                want_episodes.append(ep)
                assert not (new_state == next_state).all()
            state, pa = new_state, (0 if ep is not None else a)
    key = lambda e: (e["task"], e["episode"])
    assert sorted(episodes, key=key) == sorted(want_episodes, key=key)
    assert len(episodes) >= n and any(e["episode"] > 0 for e in episodes)
    assert all(set(e) == {"task", "episode", "prob", "score", "episode_step"} for e in episodes)
    # life losses and episode ends both occurred
    assert any(d for i in range(n) for d in got[i]["done"])


def _serve_on_cpu(pool, rounds, action=1, max_prob=0.5):
    """Drives the pool as the server would, writing every reply itself: `rounds` steps of every environment.
    -> (finished episodes, per round [rounds + 1] the reports' uniform, reset, next_state marker, frame marker)."""
    episodes, seen = [], []
    for _ in range(rounds + 1):
        ready = []
        while len(ready) < pool.num_workers:
            ready, eps = pool.wait_ready(60)
            episodes += eps
        v, E = pool.views, pool.num_envs
        seen.append(dict(uniform=v["uniform"][:E].copy(), reset=v["reset"][:E].copy(),
                         next_state=v["next_state"][:E, 0, :3, 0].copy(), frame=v["frame"][:E, 0, :3, 0].copy()))
        if len(seen) == rounds + 1:
            break
        for w in ready:
            for e in pool.env_ids(w):
                pool.views["action"][e], pool.views["max_prob"][e] = action, max_prob
        pool.reply(ready)
    return episodes, seen


def test_pool_spawns_torch_free_workers_writes_next_state_and_closes():
    import torch  # noqa: F401  (imported here, so a worker that inherited the parent's modules would show it)
    fns = [functools.partial(ScriptedEnv, i) for i in range(5)]
    seeds = [40 + i for i in range(5)]
    with S.A3CEnvWorkerPool(fns, [A] * 5, 2, seeds=seeds) as pool:
        assert pool.num_workers == 3 and [pool.env_ids(w) for w in range(3)] == [[0, 1], [2, 3], [4]]
        assert pool.exchange_bytes == S.a3c_exchange_bytes(5)
        assert len(pool.worker_info) == 3
        assert not any(i["torch"] or i["native"] for i in pool.worker_info)
        assert all(type(x["process"]).__name__ == "SpawnProcess" for x in pool._workers)
        episodes, seen = _serve_on_cpu(pool, 9)
        # each environment's uniforms come from its own stream, whatever the grouping
        for i in range(5):
            rng = np.random.RandomState(seeds[i])
            assert [s["uniform"][i] for s in seen] == [rng.random_sample() for _ in range(10)]
        # action 1: one 7-step episode each; the report after step 7 has reset set, the terminal frame (7 step calls,
        # first reset) in next_state and the second episode's first frame (7 calls, second reset) as its frame
        for k, s in enumerate(seen):
            assert list(s["reset"]) == [1 if k in (0, 7) else 0] * 5, k
        assert (seen[7]["next_state"] == [[i, 7, 1] for i in range(5)]).all()
        assert (seen[7]["frame"] == [[i, 7, 2] for i in range(5)]).all()
        # next_state is written only at an episode end: untouched before it, and kept after it
        assert not seen[6]["next_state"].any() and (seen[9]["next_state"] == seen[7]["next_state"]).all()
        key = lambda e: e["task"]
        assert sorted(episodes, key=key) == [dict(task=i, episode=0, score=7.0, episode_step=7, prob=0.5)
                                             for i in range(5)]
    assert _no_children()


def test_worker_failure_names_the_task_and_leaves_no_children():
    fns = [functools.partial(ScriptedEnv, i) for i in range(4)]
    fns[3] = functools.partial(ScriptedEnv, 3, fail_at=4)
    pool = S.A3CEnvWorkerPool(fns, [A] * 4, 2, seeds=range(4))
    try:
        with pytest.raises(RuntimeError, match="environment task 3 raised"):
            _serve_on_cpu(pool, 10)
    finally:
        pool.close()
    assert _no_children()


def test_closing_the_pool_closes_its_servers_first():
    fns = [functools.partial(ScriptedEnv, i) for i in range(2)]
    pool = S.A3CEnvWorkerPool(fns, [A] * 2, 1, seeds=range(2))
    order = []

    class Server:   # what A3CPolicyServer does with its pool
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


def test_pool_argument_checks():
    fn = functools.partial(ScriptedEnv, 0)
    with pytest.raises(ValueError, match="seeds"):
        S.A3CEnvWorkerPool([fn] * 2, [A] * 2, 1, seeds=[0])
    with pytest.raises(ValueError, match="available_action"):
        S.A3CEnvWorkerPool([fn] * 2, [A], 1, seeds=[0, 1])
    with pytest.raises(ValueError):
        S.A3CEnvWorkerPool([fn] * 257, [A] * 257, 1, seeds=range(257))
    with pytest.raises(ValueError):
        S.A3CEnvWorkerPool([], [], 1, seeds=[])
    with pytest.raises(ValueError, match="envs_per_worker"):
        S.A3CEnvWorkerPool([fn], [A], 0, seeds=[0])
    with pytest.raises(ValueError, match="cannot be pickled"):
        S.A3CEnvWorkerPool([lambda: ScriptedEnv(0)], [A], 1, seeds=[0])
    assert _no_children()


def test_server_argument_types():
    """A3CPolicyServer takes a NativeA3CPolicy and an A3CDeviceFIFOQueue; the type checks come before any device
    call."""
    class Pool:
        num_envs = 1

    with pytest.raises(TypeError, match="NativeA3CPolicy"):
        S.A3CPolicyServer(object(), object(), Pool())
    from distributed_reinforcement_learning_b200.apex_policy import NativeA3CPolicy, NativeApexPolicy
    pol = NativeA3CPolicy.__new__(NativeA3CPolicy)   # no engine behind it: never reaches the C-ABI
    with pytest.raises(TypeError, match="NativeA3CPolicy"):
        S.A3CPolicyServer(NativeApexPolicy.__new__(NativeApexPolicy), object(), Pool())
    with pytest.raises(TypeError, match="A3CDeviceFIFOQueue"):
        S.A3CPolicyServer(pol, object(), Pool())
