"""The host side of the R2D2 policy server (actor_server.py: R2D2EnvWorkerPool, R2D2PolicyServer), without a GPU: the
R2D2 exchange records against include/drl_b200.h, the shared step rule utils.r2d2_env_step against R2D2VectorActor,
the per-environment explore draws, and the worker pool's processes (spawned, torch-free, failures surfaced by task,
nothing left behind).  The replies the server's kernels would write are written by the test itself."""
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
    """84x84xC frames that encode (seed, step), a life lost every `life_every` steps and an episode end every
    `episode_len` steps; step `fail_at` raises."""

    def __init__(self, seed, life_every=3, episode_len=7, fail_at=None, channels=1):
        self.seed, self.life_every, self.episode_len, self.fail_at = seed, life_every, episode_len, fail_at
        self.channels = channels
        self.calls = 0

    def _frame(self):
        f = np.zeros((84, 84, self.channels), np.uint8)
        f[0, 0, 0], f[0, 1, 0] = self.seed, self.calls % 256
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


def test_r2d2_exchange_layout_matches_header():
    with open(os.path.join(ROOT, "include", "drl_b200.h")) as f:
        defs = {k: int(v) for k, v in re.findall(r"#define DRL_R2D2_SERVER_(\w+) (\d+)", f.read())}
    assert defs == dict(REPORT_FRAME=S.R2D2_REPORT_FRAME, REPORT_EXPLORE=S.R2D2_REPORT_EXPLORE,
                        REPORT_REWARD=S.R2D2_REPORT_REWARD, REPORT_DONE=S.R2D2_REPORT_DONE,
                        REPORT_RESET=S.R2D2_REPORT_RESET, REPORT_BYTES=S.R2D2_REPORT_BYTES,
                        REPLY_ACTION=S.R2D2_REPLY_ACTION, REPLY_Q_ACTION=S.R2D2_REPLY_Q_ACTION,
                        REPLY_BYTES=S.R2D2_REPLY_BYTES)
    # the IMPALA records' sizes, so one exchange_bytes and one block allocator serve both servers
    assert (S.R2D2_REPORT_BYTES, S.R2D2_REPLY_BYTES) == (S.REPORT_BYTES, S.REPLY_BYTES)
    # the record keeps 84x84x4 bytes for the frame at either C; every field 16-byte aligned, in order, no overlap
    offs = [S.R2D2_REPORT_FRAME, S.R2D2_REPORT_EXPLORE, S.R2D2_REPORT_REWARD, S.R2D2_REPORT_DONE, S.R2D2_REPORT_RESET]
    ends = [84 * 84 * 4, S.R2D2_REPORT_EXPLORE + 4, S.R2D2_REPORT_REWARD + 4, S.R2D2_REPORT_DONE + 1,
            S.R2D2_REPORT_RESET + 1]
    assert all(o % 16 == 0 for o in offs + [S.R2D2_REPORT_BYTES, S.R2D2_REPLY_ACTION, S.R2D2_REPLY_Q_ACTION,
                                            S.R2D2_REPLY_BYTES])
    assert all(ends[i] <= offs[i + 1] for i in range(len(offs) - 1)) and ends[-1] <= S.R2D2_REPORT_BYTES
    assert S.R2D2_REPLY_ACTION + 4 <= S.R2D2_REPLY_Q_ACTION and S.R2D2_REPLY_Q_ACTION + 4 <= S.R2D2_REPLY_BYTES


@pytest.mark.parametrize("channels", [1, 4])
def test_r2d2_exchange_views_address_the_records(channels):
    n = 5
    buf = bytearray(S.exchange_bytes(n))
    v = S.r2d2_exchange_views(buf, n, channels)
    assert v["frame"].shape == (n, 84, 84, channels)
    v["frame"][3] = 7
    v["explore"][3] = -1
    v["reward"][3], v["done"][3], v["reset"][3] = -1.0, 1, 1
    v["action"][2], v["q_action"][2] = 3, 0.5
    raw = np.frombuffer(buf, np.uint8)
    r3 = 3 * S.R2D2_REPORT_BYTES
    frame = 84 * 84 * channels
    assert (raw[r3:r3 + frame] == 7).all() and not raw[r3 + frame:r3 + S.R2D2_REPORT_EXPLORE].any()
    assert np.frombuffer(buf, np.int32, 1, r3 + S.R2D2_REPORT_EXPLORE)[0] == -1
    assert np.frombuffer(buf, np.float32, 1, r3 + S.R2D2_REPORT_REWARD)[0] == -1.0
    assert raw[r3 + S.R2D2_REPORT_DONE] == 1 and raw[r3 + S.R2D2_REPORT_RESET] == 1
    rp = n * S.R2D2_REPORT_BYTES + 2 * S.R2D2_REPLY_BYTES
    assert np.frombuffer(buf, np.int32, 1, rp + S.R2D2_REPLY_ACTION)[0] == 3
    assert np.frombuffer(buf, np.float32, 1, rp + S.R2D2_REPLY_Q_ACTION)[0] == 0.5
    # nothing else was written
    assert raw[:r3].sum() == 0 and raw[r3 + S.R2D2_REPORT_BYTES:n * S.R2D2_REPORT_BYTES].sum() == 0


class _FakeR2D2Policy:
    """NativeR2D2Policy.act's interface with a scripted rule: action = (frame[0,1,0] + previous action) % A,
    q_action = 0.25 action; h and c count the acts since the episode began.  Records the epsilons it was given."""
    max_batch, L, A = 64, 4, A

    def __init__(self):
        self.epsilons = []

    def act(self, state, previous_action, h, c, epsilon=None):
        self.epsilons.append(np.array(epsilon, np.float64))
        action = ((state[:, 0, 1, 0].astype(np.int64) + previous_action) % self.A).astype(np.int32)
        return dict(action=action, q_action=(0.25 * action).astype(np.float32), h=h + 1, c=c - 1)


class _ListQueue:
    def __init__(self):
        self.items = []

    def append_to_queue(self, task, **kw):
        self.items.append((task, kw))


def _expected_records(actions, life_every, episode_len, task):
    """What the R2D2 actor's rules give for ScriptedEnv under the recorded actions, derived without the step rule:
    per step (reward, done, previous action, steps since the episode started, epsilon of the act), and the finished
    episodes.  The life counter is only reset at an episode's end, so every step from an episode's first life loss on
    is stored as reward -1 and done; episode_step and the summed q_action run on across episodes."""
    rows, episodes = [], []
    t, episode, score, pa, lost, eps = 0, 0, 0.0, 0, False, 1.0
    total_steps, total_q = 0, 0.0
    for a in actions:
        t += 1
        total_steps += 1
        total_q += float(np.float32(0.25 * a))
        raw = float(a % 3)
        lost = lost or t % life_every == 0
        rows.append((-1.0 if lost else raw, lost, pa, t - 1, eps))
        score += raw
        pa = a
        if t >= episode_len:
            episodes.append(dict(task=task, episode=episode, score=score, epsilon=eps, episode_step=total_steps,
                                 avg_q_value=total_q / total_steps))
            t, episode, score, pa, lost = 0, episode + 1, 0.0, 0, False
            eps = 1.0 / (0.01 * episode + 1)
    return rows, episodes


def test_step_rule_gives_r2d2_vector_actor_records():
    """R2D2VectorActor (through utils.r2d2_env_step) against expectations worked out from the environments' script:
    the raw action, reward -1 and done from an episode's first life loss on, epsilon after each episode end, the
    never-reset episode_step and summed q, and the previous action, h and c back to 0 at every episode start."""
    from distributed_reinforcement_learning_b200.actor import R2D2VectorActor
    n, Sq = 3, 5
    q = _ListQueue()
    pol = _FakeR2D2Policy()
    actor = R2D2VectorActor(pol, [ScriptedEnv(i, 3 + i, 7 + i) for i in range(n)], q, Sq)
    episodes = [ep for _ in range(5) for ep in actor.run_unroll()]
    got = {i: [] for i in range(n)}
    for task, kw in q.items:
        got[task] += [(int(a), float(r), bool(d), int(pa), h, c) for a, r, d, pa, h, c in zip(
            kw["unrolled_action"], kw["unrolled_reward"], kw["unrolled_done"], kw["unrolled_previous_action"],
            kw["unrolled_previous_h"], kw["unrolled_previous_c"])]
    eps_seen = np.stack(pol.epsilons)   # [steps, n]
    want_episodes = []
    for i in range(n):
        assert len(got[i]) == 5 * Sq
        actions = [r[0] for r in got[i]]
        rows, eps = _expected_records(actions, 3 + i, 7 + i, i)
        want_episodes += eps
        for k, ((a, r, d, pa, h, c), (wr, wd, wpa, since, weps)) in enumerate(zip(got[i], rows)):
            assert (r, d, pa) == (wr, wd, wpa), (i, k)
            assert (h == since).all() and (c == -since).all()
            assert eps_seen[k, i] == weps
    key = lambda e: (e["task"], e["episode"])
    assert sorted(episodes, key=key) == sorted(want_episodes, key=key) and len(episodes) >= n
    assert any(e["episode"] > 0 for e in episodes)


@pytest.mark.parametrize("epsilon", [1.0, 0.5, 1.0 / 1.07, 0.0])
def test_explore_action_draws_as_explore_actions(epsilon):
    """A worker's per-environment draw makes the same draws from its RandomState as explore_actions makes from numpy's
    global stream seeded alike."""
    # imported here: the spawned workers import this module for ScriptedEnv, and policy_handle loads the library
    from distributed_reinforcement_learning_b200.policy_handle import explore_actions
    rng = np.random.RandomState(11)
    np.random.seed(11)
    got = [S.explore_action(rng, epsilon, A) for _ in range(200)]
    want = [int(explore_actions(epsilon, 1, A)[0]) for _ in range(200)]
    assert got == want
    assert rng.random_sample() == np.random.random_sample()   # the streams are in the same place


def _serve_on_cpu(pool, rounds, action=1, q_action=0.5):
    """Drives the pool as the server would, writing every reply itself: `rounds` steps of every environment.
    -> (finished episodes, the explore values of every report, [rounds + 1][num_envs])."""
    episodes, explores = [], []
    for _ in range(rounds + 1):
        ready = []
        while len(ready) < pool.num_workers:
            ready, eps = pool.wait_ready(60)
            episodes += eps
        explores.append(pool.views["explore"][:pool.num_envs].copy())
        if len(explores) == rounds + 1:
            break
        for w in ready:
            for e in pool.env_ids(w):
                pool.views["action"][e], pool.views["q_action"][e] = action, q_action
        pool.reply(ready)
    return episodes, np.stack(explores)


def test_pool_spawns_torch_free_workers_and_closes():
    import torch  # noqa: F401  (imported here, so a worker that inherited the parent's modules would show it)
    fns = [functools.partial(ScriptedEnv, i) for i in range(5)]
    seeds = [40 + i for i in range(5)]
    with S.R2D2EnvWorkerPool(fns, A, 2, seeds=seeds) as pool:
        assert pool.num_workers == 3 and [pool.env_ids(w) for w in range(3)] == [[0, 1], [2, 3], [4]]
        assert len(pool.worker_info) == 3
        assert not any(i["torch"] or i["native"] for i in pool.worker_info)
        assert all(type(x["process"]).__name__ == "SpawnProcess" for x in pool._workers)
        v = pool.views
        assert v["frame"].shape[1:] == (84, 84, 1)
        assert (v["reset"][:5] == 1).all()
        episodes, explores = _serve_on_cpu(pool, 12)
        # each environment's draws come from its own stream, whatever the grouping: epsilon 1 up to its episode end
        # at step 7, then 1 / 1.01
        for i in range(5):
            rng = np.random.RandomState(seeds[i])
            want = [S.explore_action(rng, 1.0 if k < 7 else 1.0 / 1.01, A) for k in range(13)]
            assert list(explores[:, i]) == want
        # action 1 throughout: raw reward 1 per step, one 7-step episode each, then steps 1..5 of the next one
        key = lambda e: e["task"]
        assert sorted(episodes, key=key) == [dict(task=i, episode=0, score=7.0, epsilon=1.0, episode_step=7,
                                                  avg_q_value=0.5) for i in range(5)]
        # the second episode lost a life at its step 3 (step 10): from then on every step is stored as -1 and done
        assert (v["reward"][:5] == -1.0).all() and (v["done"][:5] == 1).all() and (v["reset"][:5] == 0).all()
        assert (v["frame"][:5, 0, 1, 0] == 12).all() and (v["frame"][:5, 0, 0, 0] == np.arange(5)).all()
    assert _no_children()


def test_pool_writes_four_channel_frames():
    fns = [functools.partial(ScriptedEnv, i, channels=4) for i in range(2)]
    with S.R2D2EnvWorkerPool(fns, A, 1, seeds=[0, 1], channels=4) as pool:
        _serve_on_cpu(pool, 2)
        assert pool.views["frame"].shape[1:] == (84, 84, 4)
        assert (pool.views["frame"][:2, 0, 1, 0] == 2).all()
    assert _no_children()


def test_closing_the_pool_closes_its_servers_first():
    fns = [functools.partial(ScriptedEnv, i) for i in range(2)]
    pool = S.R2D2EnvWorkerPool(fns, A, 1, seeds=range(2))
    order = []

    class Server:   # what R2D2PolicyServer does with its pool
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
    fns[3] = functools.partial(ScriptedEnv, 3, fail_at=4)
    pool = S.R2D2EnvWorkerPool(fns, A, 2, seeds=range(4))
    try:
        with pytest.raises(RuntimeError, match="environment task 3 raised"):
            _serve_on_cpu(pool, 10)
    finally:
        pool.close()
    assert _no_children()


def test_env_factory_that_raises_at_start_is_reported():
    fns = [functools.partial(ScriptedEnv, 0), functools.partial(ScriptedEnv, "not a seed")]
    with pytest.raises(RuntimeError, match="environment task 1 raised"):
        S.R2D2EnvWorkerPool(fns, A, 1, seeds=[0, 1])
    assert _no_children()


def test_pool_argument_checks():
    fn = functools.partial(ScriptedEnv, 0)
    with pytest.raises(ValueError, match="seeds"):
        S.R2D2EnvWorkerPool([fn] * 2, A, 1, seeds=[0])
    with pytest.raises(ValueError):
        S.R2D2EnvWorkerPool([fn] * 257, A, 1, seeds=range(257))
    with pytest.raises(ValueError):
        S.R2D2EnvWorkerPool([], A, 1, seeds=[])
    with pytest.raises(ValueError, match="envs_per_worker"):
        S.R2D2EnvWorkerPool([fn], A, 0, seeds=[0])
    with pytest.raises(ValueError, match="channels"):
        S.R2D2EnvWorkerPool([fn], A, 1, seeds=[0], channels=3)
    with pytest.raises(ValueError, match="num_action"):
        S.R2D2EnvWorkerPool([fn], 1, 1, seeds=[0])
    with pytest.raises(ValueError, match="cannot be pickled"):
        S.R2D2EnvWorkerPool([lambda: ScriptedEnv(0)], A, 1, seeds=[0])
    assert _no_children()


def test_server_argument_types():
    """R2D2PolicyServer takes a NativeR2D2Policy and an R2D2DeviceFIFOQueue; the type checks come before any device
    call."""
    class Pool:
        num_envs, channels = 1, 1

    with pytest.raises(TypeError, match="NativeR2D2Policy"):
        S.R2D2PolicyServer(object(), object(), Pool())
    from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
    pol = NativeR2D2Policy.__new__(NativeR2D2Policy)   # no engine behind it: never reaches the C-ABI
    with pytest.raises(TypeError, match="R2D2DeviceFIFOQueue"):
        S.R2D2PolicyServer(pol, object(), Pool())


def test_r2d2_env_step_returns_the_reset_frame_at_an_episode_end():
    env = ScriptedEnv(9, life_every=2, episode_len=3)
    env.reset()
    st = S._R2D2Stats(1)
    out = [utils.r2d2_env_step(env, 2, st, 0, 1.5, task=4) for _ in range(3)]
    assert [(r, d) for _, r, d, _, _ in out] == [(2.0, False), (-1, True), (-1, True)]
    next_state, _, _, state, ep = out[-1]
    assert next_state[0, 1, 0] == 3 and state[0, 1, 0] == 3 and ep is not None   # reset() frames carry the call count
    assert ep == dict(task=4, episode=0, score=6.0, epsilon=1.0, episode_step=3, avg_q_value=1.5)
    assert st.lives == [5] and st.episode == [1] and st.epsilon == [1.0 / 1.01] and st.score == [0]
    assert st.episode_step == [3] and st.episode_q_value == [4.5]
