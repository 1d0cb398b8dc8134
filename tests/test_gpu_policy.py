"""The IMPALA policy engine on the GPU: parity with the float64 oracle, bitwise determinism (graph vs eager, repeated
calls), the GPU sampler against numpy's RandomState.choice, the device-to-device sync from a training learner, a
learner stepping while another thread acts and syncs, the error paths, and VectorActor end to end into FIFOQueue and
impala.Agent.train."""
import threading

import numpy as np
import pytest
import torch

import parity
import policy_parity as pp
from oracle import impala_torch as it
from oracle import synthetic

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu(native):
    if native.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return native


def _policy(params, max_batch=64, A=18, graph=True):
    from distributed_reinforcement_learning_b200.policy import NativePolicy
    p = NativePolicy(max_batch, num_action=A, use_cuda_graph=graph)
    p.set_params(it.flatten_params(params))
    return p


@pytest.mark.parametrize("A", [2, 18, 32])
def test_act_parity_graph_and_eager(gpu, A):
    params = it.init_params(3, torch.float32, num_action=A)
    pg, pe = _policy(params, A=A, graph=True), _policy(params, A=A, graph=False)
    try:
        for n in (1, 5, 20, 64):
            u = np.random.RandomState(n).random_sample(n)
            eg, og = pp.compare_act(pg, params, n, A, seed=100 + n, uniform=u)
            ee, oe = pp.compare_act(pe, params, n, A, seed=100 + n, uniform=u)
            for e in (eg, ee):
                assert all(v < parity.TOL for v in e.values()), (n, A, e)
            _, og2 = pp.compare_act(pg, params, n, A, seed=100 + n, uniform=u)    # replay of the captured graph
            for k in ("action", "policy", "h", "c"):
                assert og[k].shape[0] == n
                assert np.array_equal(og[k], oe[k]), (n, A, k)                       # graph == eager, bitwise
                assert np.array_equal(og[k], og2[k]), (n, A, k)                      # repeated call, bitwise
            assert np.allclose(og["policy"].sum(-1), 1.0, atol=1e-5)
            assert np.array_equal(og["max_prob"], og["policy"].max(-1))
    finally:
        pg.close()
        pe.close()


def test_sampling_matches_numpy_choice(gpu):
    A = 18
    params = it.init_params(5, torch.float32, num_action=A)
    params["actor3.w"] = params["actor3.w"] * 40.0           # peaked softmaxes: many near-zero probabilities
    pol = _policy(params, A=A)
    try:
        rows = near_zero = 0
        for call in range(32):
            seeds = call * 64 + np.arange(64)
            u = np.array([np.random.RandomState(s).random_sample() for s in seeds])
            _, out = pp.compare_act(pol, params, 64, A, seed=1000 + call, uniform=u)
            for r, s in enumerate(seeds):
                exp = np.random.RandomState(s).choice(A, p=out["policy"][r])
                assert int(out["action"][r]) == exp, (call, r)
            rows += 64
            near_zero += int((out["policy"] < 1e-6).sum())
        assert rows >= 2000 and near_zero > 0
        for uu in (0.0, 1.0 - 2.0 ** -53):                  # both ends of random_sample's range
            _, out = pp.compare_act(pol, params, 64, A, seed=77, uniform=np.full(64, uu))
            for r in range(64):
                assert int(out["action"][r]) == pp.expected_action(out["policy"][r], uu), (uu, r)
    finally:
        pol.close()


def _learner(params, A=18, B=2, T=5, graph=True):
    from distributed_reinforcement_learning_b200.learner import NativeLearner
    eng = NativeLearner(batch=B, trajectory=T, num_action=A, use_cuda_graph=graph)
    eng.set_params(it.flatten_params(params))
    return eng


def _batch(B, T, A, seed):
    b = synthetic.make_batch(B, T=T, A=A, seed=seed)
    return [b[k] for k in synthetic.TRAIN_FIELDS]


def test_sync_from_learner_with_step_in_flight(gpu):
    A, B, T = 18, 2, 5
    params = it.init_params(0, torch.float32, num_action=A)
    lrn, ctl = _learner(params), _learner(params)
    pol = _policy(it.init_params(9, torch.float32, num_action=A), max_batch=4)
    try:
        st, pa, h, c = pp.make_inputs(4, A, 3)
        outs, ctl_outs = [], []
        for s in range(4):
            args = _batch(B, T, A, 10 + s)
            lrn.stage(s % 2, *args)
            lrn.step_async(s % 2)
            pol.sync_from(lrn)                                 # snapshot = parameters AFTER the step in flight
            pol.act(st, pa, h, c)
            outs.append(lrn.wait())
            snap = pol.get_params()
            assert np.array_equal(snap, lrn.get_params())
            ctl.stage(s % 2, *args)
            ctl_outs.append(ctl.step(s % 2))
            if s == 3:
                lrn.stage(0, *_batch(B, T, A, 99))
                lrn.step(0)                                    # one more step without a sync
                assert np.array_equal(pol.get_params(), snap)
                assert not np.array_equal(lrn.get_params(), snap)
        assert outs == ctl_outs                                # the learner's scalars are untouched, bitwise
        ctl.stage(0, *_batch(B, T, A, 99))
        ctl.step(0)
        assert np.array_equal(lrn.get_params(), ctl.get_params())
    finally:
        for e in (lrn, ctl, pol):
            e.close()


def test_act_and_sync_while_the_learner_steps(gpu):
    A, B, T = 18, 4, 20
    params = it.init_params(1, torch.float32, num_action=A)
    lrn, ctl = _learner(params, B=B, T=T), _learner(params, B=B, T=T)
    pol = _policy(params, max_batch=20)
    batches = [_batch(B, T, A, 200 + s) for s in range(10)]
    st, pa, h, c = pp.make_inputs(20, A, 4)
    errors, stop = [], threading.Event()
    calls = [0]

    def learn():
        try:
            for s, args in enumerate(batches):
                lrn.stage(s % 2, *args)
                lrn.step(s % 2)
        except Exception as e:   # pragma: no cover - reported below
            errors.append(e)
        finally:
            stop.set()

    def act():
        try:
            while not stop.is_set():
                out = pol.act(st, pa, h, c)
                assert np.isfinite(out["policy"]).all()
                calls[0] += 1
                if calls[0] % 5 == 0:
                    pol.sync_from(lrn)
        except Exception as e:   # pragma: no cover - reported below
            errors.append(e)
            stop.set()
    try:
        ta, tl = threading.Thread(target=act), threading.Thread(target=learn)
        ta.start()
        tl.start()
        tl.join(300)
        ta.join(300)
        assert not errors, errors
        assert calls[0] > 0
        for s, args in enumerate(batches):
            ctl.stage(s % 2, *args)
            ctl.step(s % 2)
        assert np.array_equal(lrn.get_params(), ctl.get_params())
    finally:
        for e in (lrn, ctl, pol):
            e.close()


def test_errors(gpu):
    N = gpu
    from distributed_reinforcement_learning_b200.policy import NativePolicy
    for kw in (dict(max_batch=0), dict(max_batch=65), dict(max_batch=4, input_shape=(84, 84, 3)),
               dict(max_batch=4, input_shape=(96, 84, 4)), dict(max_batch=4, lstm_hidden_size=128)):
        with pytest.raises(N.DrlError) as ei:
            NativePolicy(**kw)
        assert ei.value.code == N.DRL_ERR_INVALID, kw
    params = it.init_params(0, torch.float32, num_action=6)
    pol = _policy(params, max_batch=4, A=6)
    lrn = _learner(it.init_params(0, torch.float32, num_action=18))
    try:
        with pytest.raises(N.DrlError) as ei:
            pol.sync_from(lrn)                                 # num_action 18 vs 6
        assert ei.value.code == N.DRL_ERR_INVALID
        st, pa, h, c = pp.make_inputs(4, 6, 1)
        u = np.full(4, 0.5)
        act = np.empty(4, np.int32)
        raw = lambda n, uu: N.lib.drl_policy_act(pol._h, n, N.ptr(st), N.ptr(pa), N.ptr(h), N.ptr(c), uu, N.ptr(act),
                                                 None, None, None)
        assert raw(0, N.ptr(u)) == N.DRL_ERR_INVALID
        assert raw(5, N.ptr(u)) == N.DRL_ERR_INVALID           # n > max_batch
        assert raw(4, None) == N.DRL_ERR_INVALID               # action without uniform
        assert b"uniform" in N.lib.drl_last_error()
        assert raw(4, N.ptr(u)) == N.DRL_OK
        # without `action`, no draws are needed
        assert N.lib.drl_policy_act(pol._h, 4, N.ptr(st), N.ptr(pa), N.ptr(h), N.ptr(c), None, None, None, None,
                                    None) == N.DRL_OK
        for bad in (dict(state=st.astype(np.float32)), dict(state=st[:, :80]), dict(state=np.concatenate([st] * 2)),
                    dict(h=h[:, :128]), dict(c=c[:3]), dict(previous_action=pa[:3]),
                    dict(previous_action=np.full(4, 6)), dict(previous_action=pa.astype(np.float32)),
                    dict(uniform=np.full(4, 1.0)), dict(uniform=np.zeros(3))):
            kw = dict(state=st, previous_action=pa, h=h, c=c, uniform=u)
            kw.update(bad)
            with pytest.raises(ValueError):
                pol.act(**kw)
        with pytest.raises(TypeError):
            pol.sync_from(object())
    finally:
        pol.close()
        lrn.close()


# ---- VectorActor end to end --------------------------------------------------------------------------------------
class SyntheticEnv:
    """Seeded uint8 frames and rewards; a life is lost at each step in `life_loss` (steps of the episode, from 1), the
    episode ends after `episode_len` steps."""

    def __init__(self, seed, episode_len, life_loss):
        self.rng = np.random.default_rng(seed)
        self.episode_len, self.life_loss = episode_len, set(life_loss)
        self.actions = []

    def reset(self):
        self.t, self.lives = 0, 5
        return self.rng.integers(0, 256, (84, 84, 4), dtype=np.uint8)

    def step(self, a):
        self.actions.append(a)
        self.t += 1
        if self.t in self.life_loss:
            self.lives -= 1
        frame = self.rng.integers(0, 256, (84, 84, 4), dtype=np.uint8)
        return frame, float(self.rng.integers(0, 3)), self.t >= self.episode_len, {"ale.lives": self.lives}


def test_vector_actor_end_to_end(gpu):
    from distributed_reinforcement_learning_b200.actor import VectorActor
    from distributed_reinforcement_learning_b200.agent import impala
    from distributed_reinforcement_learning_b200.distributed_queue import buffer_queue
    from distributed_reinforcement_learning_b200.policy import NativePolicy
    A, T, n = 18, 20, 8
    agent = impala.Agent(T, [84, 84, 4], A, 256, 0.99, 6e-4, 0.0, 1e9, 1.0, 0.05, 40.0, "abs_one", "e2e_learner",
                         "e2e_learner")
    agent.set_session(None)
    q = buffer_queue.FIFOQueue(T, [84, 84, 4], A, 2 * n, n, n, 256)
    envs = [SyntheticEnv(k, episode_len=(12 if k % 2 else 33), life_loss=(5, 9) if k < 4 else ()) for k in range(n)]
    avail = [3 + (k % 3) for k in range(n)]
    pol = NativePolicy(n, num_action=A)
    rec = []
    act = pol.act

    def recording_act(*a, **kw):
        out = act(*a, **kw)
        rec.append({k: np.array(v) for k, v in out.items()})
        return out
    pol.act = recording_act
    np.random.seed(2024)
    va = VectorActor(pol, envs, q, T, avail, learner=agent)
    try:
        for unroll in range(2):                              # host-parameter sync, then device-to-device from the learner
            rec.clear()
            va.run_unroll()
            b = q.sample_batch()
            done_at = {}                                     # (env, t) where an episode ended
            for i, env in enumerate(envs):
                for t in range(T):
                    step = unroll * T + t + 1                # global step count of env i, from 1
                    L = env.episode_len
                    if step % L == 0:
                        done_at[(i, t)] = True
            for i in range(n):
                assert np.array_equal(b.action[i], [int(r["action"][i]) for r in rec])      # un-modded
                for t in range(T):
                    assert np.array_equal(b.behavior_policy[i, t], rec[t]["policy"][i])
                    if t + 1 < T:
                        if (i, t) in done_at:
                            assert not b.previous_h[i, t + 1].any() and not b.previous_c[i, t + 1].any()
                            assert int(b.previous_action[i, t + 1]) == 0
                        else:
                            assert np.array_equal(b.previous_h[i, t + 1], rec[t]["h"][i])
                            assert np.array_equal(b.previous_c[i, t + 1], rec[t]["c"][i])
                            assert int(b.previous_action[i, t + 1]) == int(rec[t]["action"][i])
                    ep_step = (unroll * T + t) % envs[i].episode_len + 1
                    lost = i < 4 and ep_step in (5, 9)
                    assert bool(b.done[i, t]) == lost, (i, t)
                    if lost:
                        assert float(b.reward[i, t]) == -1.0
                assert envs[i].actions[unroll * T:] == [int(r["action"][i]) % avail[i] for r in rec]
            assert (b.action >= np.array(avail)[:, None]).any()
            losses = agent.train(b.state, b.reward, b.action, b.done, b.behavior_policy, b.previous_action,
                                 b.previous_h, b.previous_c)
            assert all(np.isfinite(x) for x in losses)
        agent.sync_policy(pol)                               # device to device from the trained learner
        assert np.array_equal(pol.get_params(), agent._engine.get_params())
    finally:
        pol.close()
        q.close()
        if agent._engine is not None:
            agent._engine.close()
