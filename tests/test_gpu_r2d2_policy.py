"""The R2D2 policy engine on the GPU: parity with the float64 oracle, bitwise determinism (graph vs eager, repeated
calls), the action rule (first-maximum argmax, explore rows, the host's epsilon draws), the device-to-device sync from a
training learner, a learner stepping while another thread acts and syncs, the error paths, and R2D2VectorActor end to
end into R2D2FIFOQueue and the learner loop of train_r2d2.py."""
import threading

import numpy as np
import pytest

import parity
import r2d2_policy_parity as rp
from oracle import r2d2_torch as rt

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu(native):
    if native.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return native


def _policy(params, max_batch=64, A=4, C=1, graph=True):
    from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
    p = NativeR2D2Policy(max_batch, num_action=A, input_shape=(84, 84, C), use_cuda_graph=graph)
    p.set_params(rt.flatten_params(params))
    return p


def _check_graph_eager(A, C, ns):
    params = rp.make_params(3, A, C)
    pg, pe = _policy(params, A=A, C=C, graph=True), _policy(params, A=A, C=C, graph=False)
    try:
        for n in ns:
            eg, og = rp.compare_act(pg, params, n, A, C, seed=100 + n)
            ee, oe = rp.compare_act(pe, params, n, A, C, seed=100 + n)
            for e in (eg, ee):
                assert all(v < parity.TOL for v in e.values()), (n, A, C, e)
            _, og2 = rp.compare_act(pg, params, n, A, C, seed=100 + n)      # replay of the captured graph
            for k in ("action", "q", "q_action", "h", "c"):
                assert og[k].shape[0] == n
                assert np.array_equal(og[k], oe[k]), (n, A, k)                # graph == eager, bitwise
                assert np.array_equal(og[k], og2[k]), (n, A, k)               # repeated call, bitwise
            assert np.array_equal(og["action"], np.argmax(og["q"], axis=1))  # no explore_action: every row greedy
            assert np.array_equal(og["q_action"], og["q"][np.arange(n), og["action"]])
            assert pg.last_act_ms() > 0.0
    finally:
        pg.close()
        pe.close()


@pytest.mark.parametrize("A", [2, 4, 18, 32])
def test_act_parity_graph_and_eager(gpu, A):
    _check_graph_eager(A, 1, (1, 7, 40, 64))


def test_act_parity_four_channels(gpu):
    _check_graph_eager(18, 4, (1, 40))


def test_action_rule(gpu):
    A, n = 6, 16
    params = rp.make_params(4, A)
    params["value.w"][:] = 0.0
    params["value.b"][:] = 0.0                              # q = -mean in every column: all tied
    pol = _policy(params, max_batch=n, A=A)
    try:
        _, out = rp.compare_act(pol, params, n, A, seed=5)
        assert (out["q"] == out["q"][:, :1]).all()
        assert not out["action"].any()                      # np.argmax of a tie: index 0
        params = rp.make_params(4, A)
        params["value.w"][:, 4] = params["value.w"][:, 1]
        params["value.b"][1] = params["value.b"][4] = 50.0   # columns 1 and 4: the same (largest) value
        pol.set_params(rt.flatten_params(params))
        _, out = rp.compare_act(pol, params, n, A, seed=5)
        assert (out["q"][:, 1] == out["q"][:, 4]).all() and (out["q"][:, 1] == out["q"].max(1)).all()
        assert (out["action"] == 1).all()                   # the first maximum
        explore = np.array([-1, 0, 5, -1, 3, 2, -1, 1] * 2, np.int32)
        _, out = rp.compare_act(pol, params, n, A, seed=6, explore_action=explore)
        greedy = explore < 0
        assert np.array_equal(out["action"][~greedy], explore[~greedy])
        assert np.array_equal(out["action"][greedy], np.argmax(out["q"][greedy], axis=1))
        assert np.array_equal(out["q_action"], out["q"][np.arange(n), out["action"]])
    finally:
        pol.close()


def test_epsilon_draws_follow_the_reference(gpu):
    """act(..., epsilon) consumes np.random exactly like agent/r2d2.py:181-184 applied row by row."""
    A, n = 18, 24
    params = rp.make_params(6, A)
    pol = _policy(params, max_batch=n, A=A)
    eps = np.linspace(0.0, 1.0, n)
    try:
        np.random.seed(31)
        outs = [rp.compare_act(pol, params, n, A, seed=40 + k, epsilon=eps)[1] for k in range(6)]
        after = np.random.get_state()
        np.random.seed(31)
        for out in outs:
            for r in range(n):
                if np.random.rand() > eps[r]:
                    want = np.argmax(out["q"][r])
                else:
                    want = np.random.choice(A)
                assert int(out["action"][r]) == want
        ref = np.random.get_state()
        assert np.array_equal(after[1], ref[1]) and after[2] == ref[2]
        acts = np.concatenate([o["action"] for o in outs])
        assert (acts != np.concatenate([np.argmax(o["q"], 1) for o in outs])).any()   # some rows explored
    finally:
        pol.close()


def _learner(params, A=4, C=1, B=4, S=15, bi=7, graph=True):
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET, NativeR2D2Learner
    eng = NativeR2D2Learner(batch=B, seq_len=S, burn_in=bi, num_action=A, input_shape=(84, 84, C),
                            use_cuda_graph=graph)
    eng.set_params(rt.flatten_params(params), MAIN)
    eng.set_params(rt.flatten_params(rp.make_params(11, A, C)), TARGET)
    return eng


def _batch(B, S, A, seed):
    b = rt.make_sequences(B, S=S, A=A, seed=seed)
    return (b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"], b["done"],
            b["weight"])


def test_sync_from_learner_with_step_in_flight(gpu):
    A, B, S = 4, 4, 15
    params = rp.make_params(0, A)
    lrn, ctl = _learner(params), _learner(params)
    pol = _policy(rp.make_params(9, A), max_batch=4, A=A)
    try:
        st, pa, h, c = rp.make_inputs(4, A, 1, 3)
        for s in range(4):
            args = _batch(B, S, A, 10 + s)
            lrn.stage(s % 2, *args)
            lrn.step_async(s % 2)
            pol.sync_from(lrn)                                 # snapshot = parameters AFTER the step in flight
            pol.act(st, pa, h, c)
            out, td = lrn.wait()
            snap = pol.get_params()
            assert np.array_equal(snap, lrn.get_params())
            ctl.stage(s % 2, *args)
            cout, ctd = ctl.step(s % 2)
            assert out == cout and np.array_equal(td, ctd)     # the learner's scalars are untouched, bitwise
        lrn.stage(0, *_batch(B, S, A, 99))
        lrn.step(0)                                            # one more step without a sync
        assert np.array_equal(pol.get_params(), snap)
        assert not np.array_equal(lrn.get_params(), snap)
        ctl.stage(0, *_batch(B, S, A, 99))
        ctl.step(0)
        assert np.array_equal(lrn.get_params(), ctl.get_params())
    finally:
        for e in (lrn, ctl, pol):
            e.close()


def test_act_and_sync_while_the_learner_steps(gpu):
    A, B, S = 4, 8, 20
    params = rp.make_params(1, A)
    lrn, ctl = _learner(params, B=B, S=S, bi=10), _learner(params, B=B, S=S, bi=10)
    pol = _policy(params, max_batch=40, A=A)
    batches = [_batch(B, S, A, 200 + s) for s in range(10)]
    st, pa, h, c = rp.make_inputs(40, A, 1, 4)
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
                out = pol.act(st, pa, h, c, epsilon=0.1)
                assert np.isfinite(out["q"]).all()
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
    from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
    for kw in (dict(max_batch=0), dict(max_batch=65), dict(max_batch=4, input_shape=(84, 84, 3)),
               dict(max_batch=4, input_shape=(96, 84, 1)), dict(max_batch=4, lstm_size=128),
               dict(max_batch=4, num_action=1), dict(max_batch=4, num_action=33)):
        with pytest.raises(N.DrlError) as ei:
            NativeR2D2Policy(**kw)
        assert ei.value.code == N.DRL_ERR_INVALID, kw
    A = 6
    pol = _policy(rp.make_params(0, A), max_batch=4, A=A)
    lrn_a = _learner(rp.make_params(0, 4), A=4)
    lrn_c = _learner(rp.make_params(0, A, 4), A=A, C=4)
    try:
        for lrn in (lrn_a, lrn_c):                             # num_action 4 vs 6; 4 channels vs 1
            with pytest.raises(N.DrlError) as ei:
                pol.sync_from(lrn)
            assert ei.value.code == N.DRL_ERR_INVALID
        st, pa, h, c = rp.make_inputs(4, A, 1, 1)
        act = np.empty(4, np.int32)

        def raw(n, ex=None, prev=pa):
            return N.lib.drl_r2d2_policy_act(pol._h, n, N.ptr(st), N.ptr(prev), N.ptr(h), N.ptr(c),
                                             N.ptr(ex) if ex is not None else None, N.ptr(act), None, None, None,
                                             None)
        assert raw(0) == N.DRL_ERR_INVALID
        assert raw(5) == N.DRL_ERR_INVALID                     # n > max_batch
        for bad in (-2, A):
            assert raw(4, ex=np.array([-1, 0, bad, 1], np.int32)) == N.DRL_ERR_INVALID
            assert b"explore_action" in N.lib.drl_last_error()
        assert raw(4, prev=np.array([0, 1, A, 2], np.int32)) == N.DRL_ERR_INVALID
        assert raw(4, prev=np.array([0, -1, 0, 2], np.int32)) == N.DRL_ERR_INVALID
        assert raw(4, ex=np.array([-1, 0, A - 1, -1], np.int32)) == N.DRL_OK
        assert raw(4) == N.DRL_OK
        for bad in (dict(state=st.astype(np.float32)), dict(state=st[:, :80]), dict(state=np.concatenate([st] * 2)),
                    dict(state=np.repeat(st, 4, axis=-1)), dict(h=h[:, :32]), dict(c=c[:3]),
                    dict(previous_action=pa[:3]), dict(previous_action=np.full(4, A)),
                    dict(previous_action=pa.astype(np.float32)), dict(explore_action=np.full(4, A)),
                    dict(explore_action=np.full(4, -2)), dict(explore_action=np.zeros(3, np.int32)),
                    dict(explore_action=np.zeros(4, np.float32)), dict(explore_action=np.zeros(4, np.int32),
                                                                       epsilon=0.5)):
            kw = dict(state=st, previous_action=pa, h=h, c=c)
            kw.update(bad)
            with pytest.raises(ValueError):
                pol.act(**kw)
        with pytest.raises(TypeError):
            pol.sync_from(object())
    finally:
        for e in (pol, lrn_a, lrn_c):
            e.close()


# ---- R2D2VectorActor end to end ----------------------------------------------------------------------------------
class SyntheticEnv:
    """Seeded single-channel uint8 frames and rewards; a life is lost at each step in `life_loss` (steps of the
    episode, from 1), the episode ends after `episode_len` steps."""

    def __init__(self, seed, episode_len, life_loss):
        self.rng = np.random.default_rng(seed)
        self.episode_len, self.life_loss = episode_len, set(life_loss)
        self.actions, self.rewards = [], []

    def reset(self):
        self.t, self.lives = 0, 5
        return self.rng.integers(0, 256, (84, 84, 1), dtype=np.uint8)

    def step(self, a):
        self.actions.append(a)
        self.t += 1
        if self.t in self.life_loss:
            self.lives -= 1
        frame = self.rng.integers(0, 256, (84, 84, 1), dtype=np.uint8)
        r = float(self.rng.integers(0, 3))
        self.rewards.append(r)
        return frame, r, self.t >= self.episode_len, {"ale.lives": self.lives}


def test_r2d2_vector_actor_end_to_end(gpu):
    from distributed_reinforcement_learning_b200.actor import R2D2VectorActor
    from distributed_reinforcement_learning_b200.agent import r2d2
    from distributed_reinforcement_learning_b200.distributed_queue import buffer_queue
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN
    from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
    A, S, bi, n = 4, 20, 10, 8
    agent = r2d2.Agent(S, bi, [84, 84, 1], A, 64, 0.997, 1e-4, 1e-4, 1e9, 40.0, "r2d2_e2e", "r2d2_e2e")
    agent.set_session(None)
    agent.main_to_target()
    q = buffer_queue.R2D2FIFOQueue(S, [84, 84, 1], A, 2 * n, n, n, 64)
    envs = [SyntheticEnv(k, episode_len=(12 if k % 2 else 33), life_loss=(5, 9) if k < 4 else ()) for k in range(n)]
    pol = NativeR2D2Policy(n, num_action=A)
    rec = []
    act = pol.act

    def recording_act(*a, **kw):
        out = act(*a, **kw)
        rec.append({k: np.array(v) for k, v in out.items()})
        return out
    pol.act = recording_act
    np.random.seed(2024)
    va = R2D2VectorActor(pol, envs, q, S, learner=agent)
    memory = buffer_queue.Memory(capacity=1000)
    losses = []
    try:
        for unroll in range(2):                              # host-parameter sync, then device-to-device from the learner
            rec.clear()
            finished = va.run_unroll()
            b = q.sample_batch()
            for i, env in enumerate(envs):
                L = env.episode_len
                assert np.array_equal(np.asarray(b.action[i]), [int(r["action"][i]) for r in rec])
                assert env.actions[unroll * S:] == [int(r["action"][i]) for r in rec]     # the raw action
                prev_h, prev_c = np.asarray(b.previous_h[i]), np.asarray(b.previous_c[i])
                for t in range(S):
                    step = unroll * S + t                   # global step of env i, from 0
                    ep_step = step % L + 1                  # step within its episode, from 1
                    r = rec[t]
                    assert float(r["q_action"][i]) == float(r["q"][i, r["action"][i]])
                    if t + 1 < S:
                        if ep_step == L:                    # the episode ended at t
                            assert not prev_h[t + 1].any() and not prev_c[t + 1].any()
                            assert int(b.previous_action[i][t + 1]) == 0
                        else:
                            assert np.array_equal(prev_h[t + 1], r["h"][i])
                            assert np.array_equal(prev_c[t + 1], r["c"][i])
                            assert int(b.previous_action[i][t + 1]) == int(r["action"][i])
                    lost = i < 4 and ep_step >= 5            # lives is never updated after the first life loss
                    assert bool(b.done[i][t]) == lost, (i, t)
                    assert float(b.reward[i][t]) == (-1.0 if lost else env.rewards[step])
            ends = sorted((e["task"], e["episode"]) for e in finished)
            want = sorted((i, (unroll * S + t) // envs[i].episode_len) for i in range(n) for t in range(S)
                          if (unroll * S + t + 1) % envs[i].episode_len == 0)
            assert ends == want
            for e in finished:
                assert e["epsilon"] == 1.0 / (0.01 * e["episode"] + 1)
            # the learner loop of train_r2d2.py:97-165: td error per sequence -> Memory.add -> sample -> train
            for i in range(n):
                td = agent.get_td_error(state=b.state[i], previous_action=b.previous_action[i], action=b.action[i],
                                        reward=b.reward[i], done=b.done[i], h=b.previous_h[i], c=b.previous_c[i])
                memory.add(td, [b.state[i], b.previous_action[i], b.action[i], b.reward[i], b.done[i],
                                b.previous_h[i], b.previous_c[i]])
            minibatch, idxs, weight = memory.sample(n)
            cols = list(zip(*minibatch))
            loss, td = agent.train(state=cols[0], previous_action=cols[1], action=cols[2], h=cols[5], c=cols[6],
                                   reward=cols[3], done=cols[4], weight=weight)
            for k, idx in enumerate(idxs):
                memory.update(idx, td[k])
            losses.append(loss)
        assert all(np.isfinite(x) for x in losses)
        agent.sync_policy(pol)                               # device to device from the trained learner
        assert np.array_equal(pol.get_params(), agent._engine.get_params(MAIN))
    finally:
        pol.close()
        if agent._engine is not None:
            agent._engine.close()
