"""CPU (no GPU needed): the Ape-X / A3C policy engine's C-ABI struct matches its ctypes mirror, creating an engine
without a device fails loudly (no CPU fallback) after validating its configuration, and ApexVectorActor /
A3CVectorActor keep the actor loops' bookkeeping (train_apex.py:157-231, train_a3c.py:112-183) with stub policies,
stub environments and stub queues: life losses, resets, the epsilon schedule, the two total_max_prob rules, the
LocalBuffer gate, stored vs stepped actions, and at n = 1 the reference loops' queue payloads, logs and np.random
draws."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_apex_policy_config_matches_the_c_header(native, tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    ct = native.ApexPolicyConfig
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "drl_b200.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(drl_apex_policy_config));',
             '  drl_a3c_policy* a3c = (drl_apex_policy*)0;', '  (void)a3c;']
    for fname, _ in ct._fields_:
        lines.append('  printf("%s %%zu\\n", offsetof(drl_apex_policy_config, %s));' % (fname, fname))
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


@pytest.mark.parametrize("cls", ["NativeApexPolicy", "NativeA3CPolicy"])
def test_apex_policy_create_fails_loudly_without_a_device(native, cls):
    if native.device_count() > 0:
        pytest.skip("a CUDA device is present")
    from distributed_reinforcement_learning_b200 import apex_policy
    with pytest.raises(native.DrlError) as ei:
        getattr(apex_policy, cls)(4)
    assert ei.value.code == native.DRL_ERR_CUDA and "no CPU fallback" in str(ei.value)


def test_apex_policy_create_validates_before_looking_for_a_device(native):
    from distributed_reinforcement_learning_b200.apex_policy import NativeA3CPolicy, NativeApexPolicy
    for cls in (NativeApexPolicy, NativeA3CPolicy):
        for kw in (dict(max_batch=0), dict(max_batch=65), dict(max_batch=4, input_shape=(84, 84, 1)),
                   dict(max_batch=4, input_shape=(96, 84, 4)), dict(max_batch=4, num_action=1),
                   dict(max_batch=4, num_action=33)):
            with pytest.raises(native.DrlError) as ei:
                cls(**kw)
            assert ei.value.code == native.DRL_ERR_INVALID, (cls, kw)
    for algo in (-1, 2):
        cfg = native.ApexPolicyConfig(4, 84, 84, 4, 6, algo, 0, 1)
        h = C.c_void_p()
        assert native.lib.drl_apex_policy_create(C.byref(cfg), C.byref(h)) == native.DRL_ERR_INVALID
        assert b"algo" in native.lib.drl_last_error()


# ---- stubs --------------------------------------------------------------------------------------------------------
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


def stub_row(state, previous_action, A):
    """A deterministic output row from the inputs (the stub network)."""
    s = float(state[0, 0, 0]) * 7 + float(state[0, 1, 0]) * 3 + float(previous_action)
    return np.cos(np.arange(A) * 1.7 + s).astype(np.float32)


def stub_policy_row(state, previous_action, A):
    z = np.exp(stub_row(state, previous_action, A).astype(np.float64) * 2.0)
    return (z / z.sum()).astype(np.float32)


def choice_rule(policy_row, u):
    """numpy.random.RandomState.choice(A, p=policy_row) for the uniform draw u (the engine's rule)."""
    cdf = np.cumsum(np.asarray(policy_row, np.float64))
    cdf /= cdf[-1]
    return min(int(np.searchsorted(cdf, u, side="right")), len(cdf) - 1)


class StubApexPolicy:
    """q = stub_row; the epsilon draws and action rule of NativeApexPolicy (r2d2_policy.explore_actions)."""
    A = 6

    def __init__(self, max_batch=8):
        self.max_batch = max_batch
        self.calls = []

    def act(self, state, previous_action, epsilon=None):
        from distributed_reinforcement_learning_b200.r2d2_policy import explore_actions
        n = len(state)
        q = np.stack([stub_row(state[r], previous_action[r], self.A) for r in range(n)])
        ex = explore_actions(epsilon, n, self.A)
        action = np.where(ex >= 0, ex, np.argmax(q, axis=1)).astype(np.int32)
        out = dict(action=action, q=q, q_action=q[np.arange(n), action])
        self.calls.append(dict(state=np.array(state), pa=np.array(previous_action), epsilon=np.array(epsilon), **out))
        return out


class StubA3CPolicy:
    """policy = softmax(2 stub_row); np.random.random_sample(n) and the choice rule of NativeA3CPolicy."""
    A = 6

    def __init__(self, max_batch=8):
        self.max_batch = max_batch
        self.calls = []

    def act(self, state, previous_action):
        n = len(state)
        p = np.stack([stub_policy_row(state[r], previous_action[r], self.A) for r in range(n)])
        u = np.random.random_sample(n)
        action = np.array([choice_rule(p[r], u[r]) for r in range(n)], np.int32)
        out = dict(action=action, policy=p, max_prob=p[np.arange(n), action])
        self.calls.append(dict(state=np.array(state), pa=np.array(previous_action), **out))
        return out


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


# ---- ApexVectorActor ------------------------------------------------------------------------------------------------
def test_apex_vector_actor_bookkeeping():
    from distributed_reinforcement_learning_b200.actor import ApexVectorActor
    T, units, avail = 3, 5, [6, 4, 3]
    envs = [ScriptedEnv(0, 100, []), ScriptedEnv(1, 4, [2]), ScriptedEnv(2, 7, [3, 6])]
    pol, q, lrn = StubApexPolicy(), StubQueue(), StubLearner()
    np.random.seed(5)
    va = ApexVectorActor(pol, envs, q, T, avail, learner=lrn)
    done_eps = []
    for u in range(units):
        done_eps += va.run_unroll()
        assert lrn.syncs == u + 1                       # one sync per unroll
        assert len(pol.calls) == (u + 1) * T            # one batched act per step
    steps = units * T
    # the LocalBuffer gate: a sample is pushed once a buffer holds more than 3 T transitions, then at every step
    assert [p["task"] for p in q.pushed] == [0, 1, 2] * (steps - 3 * T)
    for p in q.pushed:
        assert len(p["unrolled_state"]) == T and len(set(map(id, p["unrolled_state"]))) == T   # without replacement
    for i, env in enumerate(envs):
        raw = [int(c["action"][i]) for c in pol.calls]
        assert list(va.buffers[i].action) == raw                           # stored: the raw action
        assert env.actions == [a % avail[i] for a in raw]                 # stepped: action % available_action
    assert any(a >= avail[2] for a in va.buffers[2].action)
    # lives follow info['ale.lives'] after every step: only the step that loses a life is r = -1, done
    assert list(va.buffers[1].reward) == [0.5, -1, 0.5, 0.5] * 3 + [0.5, -1, 0.5]
    assert list(va.buffers[1].done) == [False, True, False, False] * 3 + [False, True, False]
    assert list(va.buffers[2].reward) == [0.5, 0.5, -1, 0.5, 0.5, -1, 0.5] * 2 + [0.5]
    assert list(va.buffers[0].done) == [False] * steps
    assert envs[1].resets == 4                          # the initial reset + episode ends at steps 3, 7, 11
    # after an episode end the next step starts from a reset frame and previous action 0
    assert int(pol.calls[4]["state"][1][0, 1, 0]) == 0 and int(pol.calls[4]["pa"][1]) == 0
    assert va.buffers[1].previous_action[4] == 0
    assert int(pol.calls[4]["pa"][0]) == int(pol.calls[3]["action"][0])
    # per-environment epsilon: 1 until an environment's first episode ends, then 1 / (0.05 episode + 1)
    eps = np.array([c_["epsilon"] for c_ in pol.calls])
    assert (eps[:, 0] == 1.0).all()
    for k, sl in enumerate((slice(0, 4), slice(4, 8), slice(8, 12), slice(12, 15))):
        assert (eps[sl, 1] == 1 / (k * 0.05 + 1)).all()
    assert (eps[:7, 2] == 1.0).all() and (eps[7:14, 2] == 1 / 1.05).all() and eps[14, 2] == 1 / 1.1
    # finished episodes: episode_step is reset, the summed q[action] is not
    qa = np.array([c_["q_action"] for c_ in pol.calls], np.float64)
    got = sorted((e["task"], e["episode"], e["episode_step"], e["score"], e["epsilon"]) for e in done_eps)
    assert got == [(1, 0, 4, 2.0, 1.0), (1, 1, 4, 2.0, 1 / 1.05), (1, 2, 4, 2.0, 1 / 1.1),
                   (2, 0, 7, 3.5, 1.0), (2, 1, 7, 3.5, 1 / 1.05)]
    for e in done_eps:
        i, end = e["task"], (e["episode"] + 1) * envs[e["task"]].episode_len
        assert np.isclose(e["total_max_prob"], qa[:end, i].sum() / e["episode_step"], rtol=1e-12)


def test_apex_vector_actor_rejects_bad_configurations():
    from distributed_reinforcement_learning_b200.actor import ApexVectorActor
    with pytest.raises(ValueError):
        ApexVectorActor(StubApexPolicy(), [ScriptedEnv(k, 3, []) for k in range(9)], StubQueue(), 3, [6] * 9)
    with pytest.raises(ValueError):
        ApexVectorActor(StubApexPolicy(), [ScriptedEnv(k, 3, []) for k in range(2)], StubQueue(), 3, [6])


def test_apex_vector_actor_at_n1_is_the_reference_loop():
    """At n = 1: the queue payloads, the logged values and the np.random stream equal a literal restatement of
    train_apex.py:157-231 over the same stub network and environment."""
    from distributed_reinforcement_learning_b200.actor import ApexVectorActor
    from distributed_reinforcement_learning_b200.distributed_queue import buffer_queue
    T, units, A, avail = 3, 9, StubApexPolicy.A, 4
    np.random.seed(77)
    env = ScriptedEnv(3, 5, [2, 4], blank=True)
    q = StubQueue()
    va = ApexVectorActor(StubApexPolicy(1), [env], q, T, [avail], learner=StubLearner())
    logged = []
    for _ in range(units):
        logged += va.run_unroll()
    got_state = np.random.get_state()

    # --- the reference actor, literally (actor.get_policy_and_action over the stub network) ---
    np.random.seed(77)
    renv = ScriptedEnv(3, 5, [2, 4], blank=True)

    def get_policy_and_action(state, previous_action, epsilon):
        main_q_value = stub_row(state, previous_action, A)
        if np.random.rand() > epsilon:
            action = np.argmax(main_q_value, axis=0)
        else:
            action = np.random.choice(A)
        return action, main_q_value, main_q_value[action]

    pushed, ref_logged = [], []
    local_buffer = buffer_queue.LocalBuffer(capacity=int(1e4))
    epsilon, train_step, episode, episode_step, total_max_prob = 1.0, 0, 0, 0, 0
    state = renv.reset()
    previous_action, score, lives = 0, 0, 5
    for _ in range(units):
        for _ in range(T):
            action, q_value, max_q_value = get_policy_and_action(state=state, previous_action=previous_action,
                                                                 epsilon=epsilon)
            episode_step += 1
            total_max_prob += max_q_value
            next_state, reward, done, info = renv.step(action % avail)
            score += reward
            if lives != info['ale.lives']:
                r = -1
                d = True
            else:
                r = reward
                d = False
            local_buffer.append(state=state, done=d, reward=r, next_state=next_state,
                                previous_action=previous_action, action=action)
            state = next_state
            previous_action = action
            lives = info['ale.lives']
            if len(local_buffer) > 3 * T:
                train_step += 1
                pushed.append(local_buffer.sample(T))
            if done:
                ref_logged.append((episode, score, epsilon, episode_step, total_max_prob / episode_step))
                episode_step = 0
                episode += 1
                score = 0
                lives = 5
                epsilon = 1 / (episode * 0.05 + 1)
                state = renv.reset()
                previous_action = 0
    ref_state = np.random.get_state()

    assert env.actions == [int(a) for a in renv.actions]
    assert np.array_equal(got_state[1], ref_state[1]) and got_state[2] == ref_state[2]
    assert len(q.pushed) == len(pushed) == units * T - 3 * T
    for p, ref in zip(q.pushed, pushed):
        assert p["unrolled_action"] == [int(a) for a in ref["action"]]
        assert p["unrolled_previous_action"] == [int(a) for a in ref["previous_action"]]
        assert p["unrolled_reward"] == ref["reward"] and p["unrolled_done"] == ref["done"]
        for k in range(T):
            assert np.array_equal(p["unrolled_state"][k], ref["state"][k])
            assert np.array_equal(p["unrolled_next_state"][k], ref["next_state"][k])
    assert [(e["episode"], e["score"], e["epsilon"], e["episode_step"]) for e in logged] == \
        [x[:4] for x in ref_logged]
    assert np.allclose([e["total_max_prob"] for e in logged], [x[4] for x in ref_logged], rtol=1e-6, atol=1e-6)
    assert len(logged) >= 4


# ---- A3CVectorActor -------------------------------------------------------------------------------------------------
def test_a3c_vector_actor_bookkeeping():
    from distributed_reinforcement_learning_b200.actor import A3CVectorActor
    T, units, avail = 5, 3, [6, 4, 3]
    envs = [ScriptedEnv(0, 100, []), ScriptedEnv(1, 4, [2]), ScriptedEnv(2, 7, [3, 6])]
    pol, q, lrn = StubA3CPolicy(), StubQueue(), StubLearner()
    np.random.seed(9)
    va = A3CVectorActor(pol, envs, q, T, avail, learner=lrn)
    done_eps = []
    for u in range(units):
        done_eps += va.run_unroll()
        assert lrn.syncs == u + 1
        assert len(pol.calls) == (u + 1) * T
    assert [p["task"] for p in q.pushed] == [0, 1, 2] * units        # one trajectory per environment per unroll
    for i, env in enumerate(envs):
        raw = [int(c["action"][i]) for c in pol.calls]
        stored = sum((q.pushed[3 * u + i]["unrolled_action"] for u in range(units)), [])
        assert [int(a) for a in stored] == raw
        assert env.actions == [a % avail[i] for a in raw]
    p1 = sum((q.pushed[3 * u + 1]["unrolled_reward"] for u in range(units)), [])
    assert [float(r) for r in p1] == [0.5, -1, 0.5, 0.5] * 3 + [0.5, -1, 0.5]
    d2 = sum((q.pushed[3 * u + 2]["unrolled_done"] for u in range(units)), [])
    assert [bool(d) for d in d2] == [False, False, True, False, False, True, False] * 2 + [False]
    # next_state of step t is the state of step t + 1 within an episode
    p0 = q.pushed[0]
    assert all(np.array_equal(p0["unrolled_next_state"][t], p0["unrolled_state"][t + 1]) for t in range(T - 1))
    assert int(pol.calls[4]["state"][1][0, 1, 0]) == 0 and int(pol.calls[4]["pa"][1]) == 0
    # finished episodes: score, episode_step and the summed policy[action] are all reset
    mp = np.array([c_["max_prob"] for c_ in pol.calls], np.float64)
    got = sorted((e["task"], e["episode"], e["episode_step"], e["score"]) for e in done_eps)
    assert got == [(1, 0, 4, 2.0), (1, 1, 4, 2.0), (1, 2, 4, 2.0), (2, 0, 7, 3.5), (2, 1, 7, 3.5)]
    for e in done_eps:
        L = envs[e["task"]].episode_len
        lo = e["episode"] * L
        assert np.isclose(e["prob"], mp[lo:lo + L, e["task"]].sum() / L, rtol=1e-12)


def test_a3c_vector_actor_at_n1_is_the_reference_loop():
    """At n = 1: the queue payloads, the logged values and the np.random stream equal a literal restatement of
    train_a3c.py:112-183 over the same stub network and environment."""
    from distributed_reinforcement_learning_b200 import utils
    from distributed_reinforcement_learning_b200.actor import A3CVectorActor
    T, units, A, avail = 4, 5, StubA3CPolicy.A, 4
    np.random.seed(123)
    env = ScriptedEnv(5, 6, [2, 5], blank=True)
    q = StubQueue()
    va = A3CVectorActor(StubA3CPolicy(1), [env], q, T, [avail], learner=StubLearner())
    logged = []
    for _ in range(units):
        logged += va.run_unroll()
    got_state = np.random.get_state()

    # --- the reference actor, literally (a3c.Agent.get_policy_and_action over the stub network) ---
    np.random.seed(123)
    renv = ScriptedEnv(5, 6, [2, 5], blank=True)

    def get_policy_and_action(state, previous_action):
        policy = stub_policy_row(state, previous_action, A)
        p = policy.astype(np.float64)
        action = np.random.choice(A, p=p / p.sum())
        return action, policy, policy[action]

    pushed, ref_logged = [], []
    trajectory = utils.UnrolledA3CTrajectory()
    state = renv.reset()
    previous_action = 0
    episode, score, episode_step, total_max_prob, lives = 0, 0, 0, 0, 5
    for _ in range(units):
        trajectory.initialize()
        for _ in range(T):
            action, policy, max_prob = get_policy_and_action(state=state, previous_action=previous_action)
            episode_step += 1
            total_max_prob += max_prob
            next_state, reward, done, info = renv.step(action % avail)
            score += reward
            if lives != info['ale.lives']:
                r = -1
                d = True
            else:
                r = reward
                d = False
            trajectory.append(state=state, next_state=next_state, previous_action=previous_action, action=action,
                              reward=r, done=d)
            state = next_state
            previous_action = action
            lives = info['ale.lives']
            if done:
                ref_logged.append((total_max_prob / episode_step, score, episode_step, episode))
                episode += 1
                score = 0
                episode_step = 0
                total_max_prob = 0
                state = renv.reset()
                previous_action = 0
                lives = 5
        pushed.append(trajectory.extract())
    ref_state = np.random.get_state()

    assert env.actions == [int(a) for a in renv.actions]
    assert np.array_equal(got_state[1], ref_state[1]) and got_state[2] == ref_state[2]
    assert len(q.pushed) == len(pushed) == units
    for p, ref in zip(q.pushed, pushed):
        for k in ("state", "next_state", "previous_action", "action", "reward", "done"):
            assert np.array_equal(np.asarray(p["unrolled_" + k]), ref[k]), k
    assert [(e["score"], e["episode_step"], e["episode"]) for e in logged] == [x[1:] for x in ref_logged]
    assert np.allclose([e["prob"] for e in logged], [x[0] for x in ref_logged], rtol=1e-6, atol=1e-6)
    assert len(logged) >= 2
