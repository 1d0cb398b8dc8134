"""CPU (no GPU needed): the R2D2 policy engine's C-ABI struct matches its ctypes mirror, creating an engine without a
device fails loudly (no CPU fallback), and R2D2VectorActor keeps the actor loop's bookkeeping (train_r2d2.py:167-251)
with a stub policy, stub environments and a stub queue: the per-environment epsilon schedule, the lives quirk, the
resets, and at n = 1 the reference loop's actions and np.random draws."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_r2d2_policy_config_matches_the_c_header(native, tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    ct = native.R2d2PolicyConfig
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "drl_b200.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(drl_r2d2_policy_config));']
    for fname, _ in ct._fields_:
        lines.append('  printf("%s %%zu\\n", offsetof(drl_r2d2_policy_config, %s));' % (fname, fname))
    lines += ['  return 0;', '}']
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "abi"
    subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True,
                   capture_output=True)
    got = dict(ln.rsplit(" ", 1) for ln in subprocess.run([str(exe)], check=True, capture_output=True,
                                                          text=True).stdout.splitlines())
    assert int(got["size"]) == C.sizeof(ct)
    for fname, _ in ct._fields_:
        assert int(got[fname]) == getattr(ct, fname).offset, fname


def test_r2d2_policy_create_fails_loudly_without_a_device(native):
    if native.device_count() > 0:
        pytest.skip("a CUDA device is present")
    from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
    with pytest.raises(native.DrlError) as ei:
        NativeR2D2Policy(4)
    assert ei.value.code == native.DRL_ERR_CUDA and "no CPU fallback" in str(ei.value)


def test_r2d2_policy_create_validates_before_looking_for_a_device(native):
    from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
    for kw in (dict(max_batch=0), dict(max_batch=65), dict(max_batch=4, input_shape=(84, 84, 3)),
               dict(max_batch=4, lstm_size=256), dict(max_batch=4, num_action=33)):
        with pytest.raises(native.DrlError) as ei:
            NativeR2D2Policy(**kw)
        assert ei.value.code == native.DRL_ERR_INVALID, kw


# ---- R2D2VectorActor bookkeeping with stubs ---------------------------------------------------------------------
class ScriptedEnv:
    """Frames carry (env id, step); reward = 0.5 per step; one life is lost at each step in `life_loss`; the episode
    ends after `episode_len` steps.  With `blank`, every step draws np.random.rand() as the reference's
    BlankObservation wrapper does."""

    def __init__(self, k, episode_len, life_loss, blank=False):
        self.k, self.episode_len, self.life_loss, self.blank = k, episode_len, set(life_loss), blank
        self.actions, self.resets = [], 0

    def _frame(self):
        f = np.zeros((2, 2, 1), np.uint8)
        f[0, 0, 0], f[0, 1, 0] = self.k, self.t
        return f

    def reset(self):
        self.t, self.lives = 0, 5
        self.resets += 1
        return self._frame()

    def step(self, a):
        if self.blank:
            np.random.rand()
        self.actions.append(a)
        self.t += 1
        if self.t in self.life_loss:
            self.lives -= 1
        return self._frame(), 0.5, self.t >= self.episode_len, {"ale.lives": self.lives}


def stub_q(state, previous_action, h, A):
    """A deterministic q row from the inputs (the stub network)."""
    s = float(state[0, 0, 0]) * 7 + float(state[0, 1, 0]) * 3 + float(previous_action) + float(h[0])
    return np.cos(np.arange(A) * 1.7 + s).astype(np.float32)


class StubPolicy:
    """q = stub_q; h' = c' = call + 1; the epsilon draws and action rule of NativeR2D2Policy (explore_actions)."""
    L, A = 4, 6

    def __init__(self, max_batch=8):
        self.max_batch = max_batch
        self.calls = []

    def act(self, state, previous_action, h, c, epsilon=None):
        from distributed_reinforcement_learning_b200.r2d2_policy import explore_actions
        n = len(state)
        k = len(self.calls)
        self.calls.append(dict(state=np.array(state), pa=np.array(previous_action), h=np.array(h), c=np.array(c),
                               epsilon=np.array(epsilon)))
        q = np.stack([stub_q(state[r], previous_action[r], h[r], self.A) for r in range(n)])
        ex = explore_actions(epsilon, n, self.A)
        action = np.where(ex >= 0, ex, np.argmax(q, axis=1)).astype(np.int32)
        return dict(action=action, q=q, q_action=q[np.arange(n), action], h=np.full((n, self.L), k + 1, np.float32),
                    c=np.full((n, self.L), -(k + 1), np.float32))


class StubQueue:
    def __init__(self):
        self.pushed = []

    def append_to_queue(self, **kw):
        self.pushed.append({k: (list(v) if k != "task" else v) for k, v in kw.items()})


class StubLearner:
    def __init__(self):
        self.syncs = 0

    def sync_policy(self, policy):
        self.syncs += 1


def test_r2d2_vector_actor_bookkeeping():
    from distributed_reinforcement_learning_b200.actor import R2D2VectorActor
    S = 5
    envs = [ScriptedEnv(0, 100, []), ScriptedEnv(1, 4, [2]), ScriptedEnv(2, 7, [3, 6])]
    pol, q, lrn = StubPolicy(), StubQueue(), StubLearner()
    np.random.seed(5)
    va = R2D2VectorActor(pol, envs, q, S, learner=lrn)
    done_eps = []
    for u in range(2):
        done_eps += va.run_unroll()
        assert lrn.syncs == u + 1                       # one sync per unroll
        assert len(pol.calls) == (u + 1) * S            # one batched act per step
    assert [p["task"] for p in q.pushed] == [0, 1, 2, 0, 1, 2]
    for p in q.pushed:
        assert len(p["unrolled_state"]) == S and len(p["unrolled_previous_h"]) == S
    for i, env in enumerate(envs):                      # the environment gets the raw (stored) action
        stored = q.pushed[i]["unrolled_action"] + q.pushed[3 + i]["unrolled_action"]
        assert env.actions == stored
    # env 1: life lost at its step 2 (global step 1); lives stays 5, so its steps 2..4 are all r = -1, done; the
    # episode ends after 4 steps (global step 3) and the next one starts clean
    p1 = q.pushed[1]
    assert p1["unrolled_reward"] == [0.5, -1, -1, -1, 0.5] and p1["unrolled_done"] == [False, True, True, True, False]
    assert q.pushed[4]["unrolled_done"] == [True, True, True, False, True]      # episode 2 loses a life at global 5
    assert envs[1].resets == 3                          # initial reset + episodes ended at global steps 3 and 7
    # env 2 loses lives at its steps 3 and 6 (global 2 and 5) and ends at global 6: done from global 2 to 6; the next
    # episode loses a life at its step 3 (global 9)
    assert q.pushed[2]["unrolled_done"] == [False, False, True, True, True]
    assert q.pushed[5]["unrolled_done"] == [True, True, False, False, True]
    # after the episode end at global step 3, step 4 starts from a reset frame, previous action 0 and zero state
    assert int(pol.calls[4]["state"][1][0, 1, 0]) == 0
    assert int(pol.calls[4]["pa"][1]) == 0 and not pol.calls[4]["h"][1].any() and not pol.calls[4]["c"][1].any()
    assert p1["unrolled_previous_action"][4] == 0 and not np.any(p1["unrolled_previous_h"][4])
    # other rows carry the previous step's action and state
    assert int(pol.calls[4]["pa"][0]) == q.pushed[0]["unrolled_action"][3] and float(pol.calls[4]["h"][0][0]) == 4.0
    assert float(pol.calls[4]["c"][0][0]) == -4.0
    # per-environment epsilon: 1 until an environment's first episode ends, then 1 / (0.01 episode + 1)
    eps = np.array([c_["epsilon"] for c_ in pol.calls])
    e1, e2 = 1.0 / (0.01 * 1 + 1), 1.0 / (0.01 * 2 + 1)
    assert (eps[:, 0] == 1.0).all()
    assert (eps[:4, 1] == 1.0).all() and (eps[4:8, 1] == e1).all() and (eps[8:, 1] == e2).all()
    assert (eps[:7, 2] == 1.0).all() and (eps[7:, 2] == e1).all()
    # finished episodes: env 1 twice, env 2 once; episode_step and the summed q keep counting across episodes
    got = sorted((e["task"], e["episode"], e["episode_step"], e["score"], e["epsilon"]) for e in done_eps)
    assert got == [(1, 0, 4, 2.0, 1.0), (1, 1, 8, 2.0, e1), (2, 0, 7, 3.5, 1.0)]


def test_r2d2_vector_actor_rejects_too_many_envs():
    from distributed_reinforcement_learning_b200.actor import R2D2VectorActor
    with pytest.raises(ValueError):
        R2D2VectorActor(StubPolicy(), [ScriptedEnv(k, 3, []) for k in range(9)], StubQueue(), 3)


def test_r2d2_vector_actor_at_n1_is_the_reference_loop():
    """At n = 1: the actions, the stored trajectory and the np.random stream equal a literal restatement of
    train_r2d2.py:186-240 over the same stub network and environment."""
    from distributed_reinforcement_learning_b200.actor import R2D2VectorActor
    S, units, A, L = 6, 4, StubPolicy.A, StubPolicy.L
    np.random.seed(77)
    env = ScriptedEnv(3, 5, [2, 4], blank=True)
    q = StubQueue()
    va = R2D2VectorActor(StubPolicy(1), [env], q, S, learner=StubLearner())
    logged = []
    for _ in range(units):
        logged += va.run_unroll()
    got_state = np.random.get_state()

    # --- the reference actor, literally (agent.get_action over the stub network) ---
    np.random.seed(77)
    renv = ScriptedEnv(3, 5, [2, 4], blank=True)
    calls = [0]

    def get_action(state, h, c, previous_action, epsilon):
        q_value = stub_q(state, previous_action, h, A)
        h2 = np.full(L, calls[0] + 1, np.float32)
        c2 = np.full(L, -(calls[0] + 1), np.float32)
        calls[0] += 1
        if np.random.rand() > epsilon:
            action = np.argmax(q_value)
        else:
            action = np.random.choice(A)
        return action, q_value[action], h2, c2

    pushed, ref_logged = [], []
    episode, epsilon, score, lives, episode_step, episode_q_value = 0, 1, 0, 5, 0, 0
    state = renv.reset()
    previous_action = 0
    previous_h = np.zeros(L)
    previous_c = np.zeros(L)
    for _ in range(units):
        traj = []
        for _ in range(S):
            action, q_value, h, c = get_action(state=state, h=previous_h, c=previous_c,
                                               previous_action=previous_action, epsilon=epsilon)
            episode_q_value += q_value
            episode_step += 1
            next_state, reward, done, info = renv.step(action)
            score += reward
            if lives != info['ale.lives']:
                r = -1
                d = True
            else:
                r = reward
                d = False
            traj.append((state, previous_action, action, r, d, previous_h, previous_c))
            state = next_state
            previous_action = action
            previous_c = c
            previous_h = h
            if done:
                ref_logged.append((episode, score, epsilon, episode_step, episode_q_value / episode_step))
                episode += 1
                score = 0
                epsilon = 1.0 / (0.01 * episode + 1)
                state = renv.reset()
                previous_action = 0
                previous_h = np.zeros(L)
                previous_c = np.zeros(L)
                done = False
                lives = 5
        pushed.append(traj)
    ref_state = np.random.get_state()

    assert env.actions == [int(a) for a in renv.actions]
    assert np.array_equal(got_state[1], ref_state[1]) and got_state[2] == ref_state[2]
    assert any(a != int(np.argmax(stub_q(np.zeros((2, 2, 1)), 0, np.zeros(1), A))) for a in env.actions)
    for p, traj in zip(q.pushed, pushed):
        assert p["unrolled_action"] == [int(t[2]) for t in traj]
        assert p["unrolled_previous_action"] == [int(t[1]) for t in traj]
        assert p["unrolled_reward"] == [t[3] for t in traj] and p["unrolled_done"] == [t[4] for t in traj]
        for k in range(S):
            assert np.array_equal(p["unrolled_state"][k], traj[k][0])
            assert np.array_equal(p["unrolled_previous_h"][k], traj[k][5])
            assert np.array_equal(p["unrolled_previous_c"][k], traj[k][6])
    assert [(e["episode"], e["score"], e["epsilon"], e["episode_step"]) for e in logged] == \
        [x[:4] for x in ref_logged]
    assert np.allclose([e["avg_q_value"] for e in logged], [x[4] for x in ref_logged], rtol=1e-6)
