"""CPU (no GPU needed): the policy engine's C-ABI struct matches its ctypes mirror, creating an engine without a device
fails loudly (no CPU fallback), and VectorActor keeps the actor loop's bookkeeping (train_impala.py:117-194) with a stub
policy and a stub queue: life loss, episode resets, modded env action vs stored action, one sync per unroll, task ids."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_policy_config_matches_the_c_header(native, tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    ct = native.PolicyConfig
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "drl_b200.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(drl_policy_config));']
    for fname, _ in ct._fields_:
        lines.append('  printf("%s %%zu\\n", offsetof(drl_policy_config, %s));' % (fname, fname))
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


def test_policy_create_fails_loudly_without_a_device(native):
    if native.device_count() > 0:
        pytest.skip("a CUDA device is present")
    from distributed_reinforcement_learning_b200.policy import NativePolicy
    with pytest.raises(native.DrlError) as ei:
        NativePolicy(4)
    assert ei.value.code == native.DRL_ERR_CUDA and "no CPU fallback" in str(ei.value)


def test_policy_create_validates_before_looking_for_a_device(native):
    from distributed_reinforcement_learning_b200.policy import NativePolicy
    for kw in (dict(max_batch=0), dict(max_batch=65), dict(max_batch=4, input_shape=(84, 84, 1)),
               dict(max_batch=4, lstm_hidden_size=128), dict(max_batch=4, num_action=33)):
        with pytest.raises(native.DrlError) as ei:
            NativePolicy(**kw)
        assert ei.value.code == native.DRL_ERR_INVALID, kw


# ---- VectorActor bookkeeping with stubs ---------------------------------------------------------------------------
class ScriptedEnv:
    """Frames carry (env id, step); reward = 0.5 per step; one life is lost at each step in `life_loss`; the episode
    ends after `episode_len` steps."""

    def __init__(self, k, episode_len, life_loss):
        self.k, self.episode_len, self.life_loss = k, episode_len, set(life_loss)
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
        self.actions.append(a)
        self.t += 1
        if self.t in self.life_loss:
            self.lives -= 1
        return self._frame(), 0.5, self.t >= self.episode_len, {"ale.lives": self.lives}


class StubPolicy:
    """Action = 7 + row + call (always >= available_action, so the modulo shows); h = c = call + 1."""
    max_batch, L, A = 8, 4, 12

    def __init__(self):
        self.calls = []

    def act(self, state, previous_action, h, c):
        n = len(state)
        k = len(self.calls)
        self.calls.append(dict(state=np.array(state), pa=np.array(previous_action), h=np.array(h), c=np.array(c)))
        pol = np.full((n, self.A), 1.0 / self.A, np.float32)
        return dict(action=(7 + np.arange(n) + k).astype(np.int32), policy=pol, max_prob=pol.max(-1),
                    h=np.full((n, self.L), k + 1, np.float32), c=np.full((n, self.L), -(k + 1), np.float32))


class StubQueue:
    def __init__(self):
        self.pushed = []

    def append_to_queue(self, **kw):
        self.pushed.append(kw)


class StubLearner:
    def __init__(self):
        self.syncs = 0

    def sync_policy(self, policy):
        self.syncs += 1


def test_vector_actor_bookkeeping():
    from distributed_reinforcement_learning_b200.actor import VectorActor
    T = 5
    envs = [ScriptedEnv(0, 100, []), ScriptedEnv(1, 4, [2]), ScriptedEnv(2, 7, [3, 6])]
    avail = [6, 4, 3]
    pol, q, lrn = StubPolicy(), StubQueue(), StubLearner()
    va = VectorActor(pol, envs, q, T, avail, learner=lrn)
    done_eps = []
    for u in range(2):
        done_eps += va.run_unroll()
        assert lrn.syncs == u + 1                       # one sync per unroll
        assert len(pol.calls) == (u + 1) * T            # one batched act per step
    assert [p["task"] for p in q.pushed] == [0, 1, 2, 0, 1, 2]
    for i, env in enumerate(envs):                      # env sees the modded action
        assert env.actions == [(7 + i + k) % avail[i] for k in range(2 * T)]
    for j, p in enumerate(q.pushed):
        i, u = p["task"], j // 3
        assert p["unrolled_action"] == [7 + i + k for k in range(u * T, (u + 1) * T)]   # stored un-modded
        assert len(p["unrolled_state"]) == T and len(p["unrolled_behavior_policy"]) == T
    # env 1: life lost at its step 2 (global step 1) -> r = -1, d = True; the episode ends after 4 steps (global step 3)
    p1 = q.pushed[1]
    assert p1["unrolled_reward"] == [0.5, -1.0, 0.5, 0.5, 0.5] and p1["unrolled_done"] == [False, True, False, False, False]
    assert envs[1].resets == 3                          # initial reset + episodes ended at global steps 3 and 7
    # after the episode end at global step 3, step 4 starts from a reset frame, previous action 0 and zero state
    assert int(pol.calls[4]["state"][1][0, 1, 0]) == 0
    assert int(pol.calls[4]["pa"][1]) == 0 and not pol.calls[4]["h"][1].any() and not pol.calls[4]["c"][1].any()
    assert p1["unrolled_previous_action"][4] == 0 and not np.any(p1["unrolled_previous_h"][4])
    # other rows carry the previous step's action and state
    assert int(pol.calls[4]["pa"][0]) == 7 + 0 + 3 and float(pol.calls[4]["h"][0][0]) == 4.0
    assert float(pol.calls[4]["c"][0][0]) == -4.0
    # env 2 loses lives at its steps 3 and 6 (global 2 and 5), ends its episode at global step 6 and loses a life at
    # step 3 of the next episode (global 9)
    assert q.pushed[2]["unrolled_done"] == [False, False, True, False, False]
    assert q.pushed[5]["unrolled_done"] == [True, False, False, False, True]
    assert q.pushed[5]["unrolled_reward"][0] == -1.0
    # finished episodes: env 1 twice (4 steps each), env 2 once (7 steps); scores keep the raw rewards
    got = sorted((e["task"], e["episode"], e["episode_step"], e["score"]) for e in done_eps)
    assert got == [(1, 0, 4, 2.0), (1, 1, 4, 2.0), (2, 0, 7, 3.5)]
    assert all(abs(e["prob"] - 1.0 / 12) < 1e-7 for e in done_eps)


def test_vector_actor_rejects_too_many_envs():
    from distributed_reinforcement_learning_b200.actor import VectorActor
    envs = [ScriptedEnv(k, 3, []) for k in range(9)]
    with pytest.raises(ValueError):
        VectorActor(StubPolicy(), envs, StubQueue(), 3, [4] * 9)
    with pytest.raises(ValueError):
        VectorActor(StubPolicy(), envs[:2], StubQueue(), 3, [4])
