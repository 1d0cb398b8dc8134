"""The Ape-X / A3C policy engine on the GPU: q / policy parity with the float64 oracle, bitwise determinism (graph vs
eager, repeated calls), the action rules (first-maximum argmax, explore rows and the host's epsilon draws for Ape-X;
numpy's choice for A3C, with uniforms on the cdf boundaries), the device-to-device sync from a training learner, a
learner stepping while another thread acts and syncs, the error paths, and ApexVectorActor / A3CVectorActor end to
end through the learner loops of train_apex.py and train_a3c.py."""
import threading

import numpy as np
import pytest

import apex_policy_parity as ap
import parity

pytestmark = pytest.mark.gpu

APEX, A3C = ap.APEX, ap.A3C


@pytest.fixture(scope="module")
def gpu(native):
    if native.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return native


def _policy(params, algo, max_batch=64, A=4, graph=True):
    from distributed_reinforcement_learning_b200.apex_policy import NativeA3CPolicy, NativeApexPolicy
    cls = NativeApexPolicy if algo == APEX else NativeA3CPolicy
    p = cls(max_batch, num_action=A, use_cuda_graph=graph)
    p.set_params(ap.flatten_params(params))
    return p


def _act_kw(algo, n, seed):
    if algo == APEX:
        return {}
    return dict(uniform=np.random.RandomState(seed).random_sample(n))


@pytest.mark.parametrize("algo", [APEX, A3C])
@pytest.mark.parametrize("A", [2, 4, 18, 32])
def test_act_parity_graph_and_eager(gpu, algo, A):
    params = ap.make_params(3, A, algo)
    pg, pe = _policy(params, algo, A=A, graph=True), _policy(params, algo, A=A, graph=False)
    out_key = "q" if algo == APEX else "policy"
    sel_key = "q_action" if algo == APEX else "max_prob"
    try:
        for n in (1, 7, 20, 64):
            kw = _act_kw(algo, n, 50 + n)
            eg, og = ap.compare_act(pg, params, n, A, seed=100 + n, **kw)
            ee, oe = ap.compare_act(pe, params, n, A, seed=100 + n, **kw)
            for e in (eg, ee):
                assert all(v < parity.TOL for v in e.values()), (n, A, algo, e)
            _, og2 = ap.compare_act(pg, params, n, A, seed=100 + n, **kw)      # replay of the captured graph
            for k in ("action", out_key, sel_key):
                assert og[k].shape[0] == n
                assert np.array_equal(og[k], oe[k]), (n, A, k)                # graph == eager, bitwise
                assert np.array_equal(og[k], og2[k]), (n, A, k)               # repeated call, bitwise
            assert np.array_equal(og[sel_key], og[out_key][np.arange(n), og["action"]])
            if algo == APEX:
                assert np.array_equal(og["action"], np.argmax(og["q"], axis=1))   # no explore_action: greedy
            else:
                assert np.allclose(og["policy"].sum(1), 1.0, atol=1e-5)
                want = [ap.expected_action(og["policy"][r], kw["uniform"][r]) for r in range(n)]
                assert og["action"].tolist() == want
            assert pg.last_act_ms() > 0.0
    finally:
        pg.close()
        pe.close()


def test_apex_action_rule(gpu):
    A, n = 6, 16
    params = ap.make_params(4, A)
    params["value3.w"][:] = 0.0
    params["value3.b"][:] = 0.0                             # q = -mean in every column: all tied
    pol = _policy(params, APEX, max_batch=n, A=A)
    try:
        _, out = ap.compare_act(pol, params, n, A, seed=5)
        assert (out["q"] == out["q"][:, :1]).all()
        assert not out["action"].any()                      # np.argmax of a tie: index 0
        params = ap.make_params(4, A)
        params["value3.w"][:, 4] = params["value3.w"][:, 1]
        params["value3.b"][1] = params["value3.b"][4] = 50.0   # columns 1 and 4: the same (largest) value
        pol.set_params(ap.flatten_params(params))
        _, out = ap.compare_act(pol, params, n, A, seed=5)
        assert (out["q"][:, 1] == out["q"][:, 4]).all() and (out["q"][:, 1] == out["q"].max(1)).all()
        assert (out["action"] == 1).all()                   # the first maximum
        explore = np.array([-1, 0, 5, -1, 3, 2, -1, 1] * 2, np.int32)
        _, out = ap.compare_act(pol, params, n, A, seed=6, explore_action=explore)
        greedy = explore < 0
        assert np.array_equal(out["action"][~greedy], explore[~greedy])
        assert np.array_equal(out["action"][greedy], np.argmax(out["q"][greedy], axis=1))
        assert np.array_equal(out["q_action"], out["q"][np.arange(n), out["action"]])
    finally:
        pol.close()


def test_apex_epsilon_draws_follow_the_reference(gpu):
    """act(..., epsilon) consumes np.random exactly like agent/apex.py:97-101 applied row by row."""
    A, n = 18, 24
    params = ap.make_params(6, A)
    pol = _policy(params, APEX, max_batch=n, A=A)
    eps = np.linspace(0.0, 1.0, n)
    try:
        np.random.seed(31)
        outs = [ap.compare_act(pol, params, n, A, seed=40 + k, epsilon=eps)[1] for k in range(6)]
        after = np.random.get_state()
        np.random.seed(31)
        for out in outs:
            for r in range(n):
                if np.random.rand() > eps[r]:
                    want = np.argmax(out["q"][r], axis=0)
                else:
                    want = np.random.choice(A)
                assert int(out["action"][r]) == want
        ref = np.random.get_state()
        assert np.array_equal(after[1], ref[1]) and after[2] == ref[2]
        acts = np.concatenate([o["action"] for o in outs])
        assert (acts != np.concatenate([np.argmax(o["q"], 1) for o in outs])).any()   # some rows explored
    finally:
        pol.close()


def test_a3c_actions_follow_numpy_choice(gpu):
    """The default uniforms are np.random.random_sample(n): row by row the same stream and the same action as
    np.random.RandomState(s).choice(A, p=policy_row)."""
    A, n = 18, 64
    params = ap.make_params(8, A, A3C)
    pol = _policy(params, A3C, max_batch=n, A=A)
    try:
        for s in range(4):
            np.random.seed(s)
            _, out = ap.compare_act(pol, params, n, A, seed=60 + s)
            rs = np.random.RandomState(s)
            want = [int(rs.choice(A, p=out["policy"][r])) for r in range(n)]
            assert out["action"].tolist() == want
            assert np.array_equal(np.random.get_state()[1], rs.get_state()[1])
            assert np.array_equal(out["max_prob"], out["policy"][np.arange(n), out["action"]])
    finally:
        pol.close()


def test_a3c_uniform_on_cdf_boundaries(gpu):
    """u exactly on cdf[k] takes k + 1 (searchsorted side='right'); u = 0 and u = 1 - 2^-53 stay in range."""
    A, n = 6, 8
    params = ap.make_params(9, A, A3C)
    pol = _policy(params, A3C, max_batch=n, A=A)
    try:
        st, pa = ap.make_inputs(n, A, 11)
        base = pol.act(st, pa, uniform=np.full(n, 0.5))["policy"]
        cdf = np.cumsum(base.astype(np.float64), axis=1)
        cdf /= cdf[:, -1:]
        for k in range(A - 1):
            u = cdf[:, k].copy()
            out = pol.act(st, pa, uniform=u)
            assert np.array_equal(out["policy"], base)
            want = [ap.expected_action(base[r], u[r]) for r in range(n)]
            assert out["action"].tolist() == want
            assert all(w == k + 1 for w, p in zip(want, base[:, k + 1]) if p > 0)
            below = np.nextafter(u, 0.0)                     # one ulp below the boundary: still k
            assert pol.act(st, pa, uniform=below)["action"].tolist() == [ap.expected_action(base[r], below[r])
                                                                          for r in range(n)]
        assert not pol.act(st, pa, uniform=np.zeros(n))["action"].any() or (base[:, 0] == 0).any()
        top = pol.act(st, pa, uniform=np.full(n, 1.0 - 2.0 ** -53))["action"]
        assert top.tolist() == [ap.expected_action(base[r], 1.0 - 2.0 ** -53) for r in range(n)]
        assert (top <= A - 1).all()
    finally:
        pol.close()


# ---- sync from a training learner -----------------------------------------------------------------------------------
def _learner(params, algo, A=4, B=4, graph=True):
    if algo == APEX:
        from distributed_reinforcement_learning_b200.apex_learner import MAIN, TARGET, NativeApexLearner
        eng = NativeApexLearner(batch=B, num_action=A, use_cuda_graph=graph)
        eng.set_params(ap.flatten_params(params), MAIN)
        eng.set_params(ap.flatten_params(ap.make_params(11, A)), TARGET)
    else:
        from distributed_reinforcement_learning_b200.a3c_learner import NativeA3CLearner
        eng = NativeA3CLearner(batch=B, num_action=A, use_cuda_graph=graph)
        eng.set_params(ap.flatten_params(params))
    return eng


def _main(lrn, algo):
    if algo == APEX:
        from distributed_reinforcement_learning_b200.apex_learner import MAIN
        return lrn.get_params(MAIN)
    return lrn.get_params()


def _batch(B, A, seed, algo):
    from oracle import apex_torch as ax
    t = ax.make_transitions(B, A=A, seed=seed)
    args = [t["state"], t["next_state"], t["previous_action"], t["action"], t["reward"], t["done"]]
    return args + [t["is_weight"]] if algo == APEX else args


def _step(lrn, algo, slot, args, wait=True):
    lrn.stage(slot, *args)
    if not wait:
        lrn.step_async(slot)
        return None
    out = lrn.step(slot)
    return out


@pytest.mark.parametrize("algo", [APEX, A3C])
def test_sync_from_learner_with_step_in_flight(gpu, algo):
    A, B = 4, 4
    params = ap.make_params(0, A, algo)
    lrn, ctl = _learner(params, algo), _learner(params, algo)
    pol = _policy(ap.make_params(9, A, algo), algo, max_batch=4, A=A)
    try:
        st, pa = ap.make_inputs(4, A, 3)
        kw = _act_kw(algo, 4, 1)
        for s in range(4):
            args = _batch(B, A, 10 + s, algo)
            _step(lrn, algo, s % 2, args, wait=False)
            pol.sync_from(lrn)                                 # snapshot = parameters AFTER the step in flight
            pol.act(st, pa, **kw)
            out = lrn.wait()
            snap = pol.get_params()
            assert np.array_equal(snap, _main(lrn, algo))
            cout = _step(ctl, algo, s % 2, args)
            if algo == APEX:
                assert out[0] == cout[0] and np.array_equal(out[1], cout[1])   # scalars and priorities, bitwise
            else:
                assert out == cout
        _step(lrn, algo, 0, _batch(B, A, 99, algo))            # one more step without a sync
        assert np.array_equal(pol.get_params(), snap)
        assert not np.array_equal(_main(lrn, algo), snap)
        _step(ctl, algo, 0, _batch(B, A, 99, algo))
        assert np.array_equal(_main(lrn, algo), _main(ctl, algo))
    finally:
        for e in (lrn, ctl, pol):
            e.close()


@pytest.mark.parametrize("algo", [APEX, A3C])
def test_act_and_sync_while_the_learner_steps(gpu, algo):
    A, B = 4, 32
    params = ap.make_params(1, A, algo)
    lrn, ctl = _learner(params, algo, B=B), _learner(params, algo, B=B)
    pol = _policy(params, algo, max_batch=40, A=A)
    batches = [_batch(B, A, 200 + s, algo) for s in range(10)]
    st, pa = ap.make_inputs(40, A, 4)
    errors, stop = [], threading.Event()
    calls = [0]

    def learn():
        try:
            for s, args in enumerate(batches):
                _step(lrn, algo, s % 2, args)
        except Exception as e:   # pragma: no cover - reported below
            errors.append(e)
        finally:
            stop.set()

    def act():
        try:
            while not stop.is_set():
                out = pol.act(st, pa, epsilon=0.1) if algo == APEX else pol.act(st, pa)
                assert np.isfinite(out["q" if algo == APEX else "policy"]).all()
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
            _step(ctl, algo, s % 2, args)
        assert np.array_equal(_main(lrn, algo), _main(ctl, algo))
    finally:
        for e in (lrn, ctl, pol):
            e.close()


def test_errors(gpu):
    N = gpu
    from distributed_reinforcement_learning_b200.apex_policy import NativeA3CPolicy, NativeApexPolicy
    for cls in (NativeApexPolicy, NativeA3CPolicy):
        for kw in (dict(max_batch=0), dict(max_batch=65), dict(max_batch=4, input_shape=(84, 84, 1)),
                   dict(max_batch=4, input_shape=(96, 84, 4)), dict(max_batch=4, num_action=1),
                   dict(max_batch=4, num_action=33)):
            with pytest.raises(N.DrlError) as ei:
                cls(**kw)
            assert ei.value.code == N.DRL_ERR_INVALID, kw
    A = 6
    px = _policy(ap.make_params(0, A), APEX, max_batch=4, A=A)
    pc = _policy(ap.make_params(0, A, A3C), A3C, max_batch=4, A=A)
    lx, lx4 = _learner(ap.make_params(0, A), APEX, A=A), _learner(ap.make_params(0, 4), APEX, A=4)
    lc, lc4 = _learner(ap.make_params(0, A, A3C), A3C, A=A), _learner(ap.make_params(0, 4, A3C), A3C, A=4)
    try:
        px.sync_from(lx)
        pc.sync_from(lc)
        for pol, lrn in ((px, lx4), (pc, lc4)):                # num_action 4 vs 6
            with pytest.raises(N.DrlError) as ei:
                pol.sync_from(lrn)
            assert ei.value.code == N.DRL_ERR_INVALID
        for pol, lrn in ((px, lc), (pc, lx)):                  # the other family's learner
            assert N.lib.drl_apex_policy_sync_from_learner(pol._h, lrn._h) == N.DRL_ERR_INVALID
            assert b"A3C" in N.lib.drl_last_error()
            with pytest.raises(TypeError):
                pol.sync_from(lrn)
        with pytest.raises(TypeError):
            px.sync_from(object())
        assert N.lib.drl_apex_policy_sync_from_learner(px._h, None) == N.DRL_ERR_INVALID
        st, pa = ap.make_inputs(4, A, 1)
        act, q, qa = np.empty(4, np.int32), np.empty((4, A), np.float32), np.empty(4, np.float32)
        u = np.full(4, 0.5)

        def rx(n, ex=None, prev=pa, state=st, h=px):
            return N.lib.drl_apex_policy_act(h._h, n, N.ptr(state) if state is not None else None,
                                             N.ptr(prev) if prev is not None else None,
                                             N.ptr(ex) if ex is not None else None, N.ptr(act), N.ptr(q), N.ptr(qa))

        def rc(n, uni=u, prev=pa, state=st, h=pc):
            return N.lib.drl_a3c_policy_act(h._h, n, N.ptr(state) if state is not None else None,
                                            N.ptr(prev) if prev is not None else None,
                                            N.ptr(uni) if uni is not None else None, N.ptr(act), N.ptr(q), N.ptr(qa))
        assert rx(4, h=pc) == N.DRL_ERR_INVALID and b"drl_a3c_policy_act" in N.lib.drl_last_error()
        assert rc(4, h=px) == N.DRL_ERR_INVALID and b"drl_apex_policy_act" in N.lib.drl_last_error()
        for r in (rx, rc):
            assert r(0) == N.DRL_ERR_INVALID
            assert r(5) == N.DRL_ERR_INVALID                   # n > max_batch
            assert r(4, prev=np.array([0, 1, A, 2], np.int32)) == N.DRL_ERR_INVALID
            assert r(4, prev=np.array([0, -1, 0, 2], np.int32)) == N.DRL_ERR_INVALID
            assert r(4, prev=None) == N.DRL_ERR_INVALID
            assert r(4, state=None) == N.DRL_ERR_INVALID
            assert r(4) == N.DRL_OK
        for bad in (-2, A):
            assert rx(4, ex=np.array([-1, 0, bad, 1], np.int32)) == N.DRL_ERR_INVALID
            assert b"explore_action" in N.lib.drl_last_error()
        assert rx(4, ex=np.array([-1, 0, A - 1, -1], np.int32)) == N.DRL_OK
        for bad in (-0.25, 1.0, np.nan, np.inf):
            assert rc(4, uni=np.array([0.1, bad, 0.2, 0.3])) == N.DRL_ERR_INVALID
            assert b"uniform" in N.lib.drl_last_error()
        assert rc(4, uni=None) == N.DRL_ERR_INVALID
        assert rc(4, uni=np.array([0.0, 0.5, 1.0 - 2.0 ** -53, 0.9])) == N.DRL_OK
        for bad in (dict(state=st.astype(np.float32)), dict(state=st[:, :80]), dict(state=np.concatenate([st] * 17)),
                    dict(state=st[..., :1]), dict(previous_action=pa[:3]), dict(previous_action=np.full(4, A)),
                    dict(previous_action=pa.astype(np.float32))):
            for pol in (px, pc):
                kw = dict(state=st, previous_action=pa)
                kw.update(bad)
                with pytest.raises(ValueError):
                    pol.act(**kw)
        for bad in (dict(explore_action=np.full(4, A)), dict(explore_action=np.full(4, -2)),
                    dict(explore_action=np.zeros(3, np.int32)), dict(explore_action=np.zeros(4, np.float32)),
                    dict(explore_action=np.zeros(4, np.int32), epsilon=0.5)):
            with pytest.raises(ValueError):
                px.act(st, pa, **bad)
        for bad in (np.full(4, 1.0), np.full(4, -0.1), np.zeros(3), np.zeros(4, np.int64), np.full(4, np.nan)):
            with pytest.raises(ValueError):
                pc.act(st, pa, uniform=bad)
    finally:
        for e in (px, pc, lx, lx4, lc, lc4):
            e.close()


# ---- the vector actors end to end ---------------------------------------------------------------------------------
class SyntheticEnv:
    """Seeded uint8 frames [84, 84, 4] and rewards; a life is lost at each step in `life_loss` (steps of the episode,
    from 1), the episode ends after `episode_len` steps."""

    def __init__(self, seed, episode_len, life_loss):
        self.rng = np.random.default_rng(seed)
        self.episode_len, self.life_loss = episode_len, set(life_loss)
        self.actions, self.rewards = [], []

    def reset(self):
        self.t, self.lives = 0, 5
        return self.rng.integers(0, 256, (84, 84, 4), dtype=np.uint8)

    def step(self, a):
        self.actions.append(a)
        self.t += 1
        if self.t in self.life_loss:
            self.lives -= 1
        frame = self.rng.integers(0, 256, (84, 84, 4), dtype=np.uint8)
        r = float(self.rng.integers(0, 3))
        self.rewards.append(r)
        return frame, r, self.t >= self.episode_len, {"ale.lives": self.lives}


def _recording(pol):
    rec = []
    act = pol.act

    def recording_act(*a, **kw):
        out = act(*a, **kw)
        rec.append({k: np.array(v) for k, v in out.items()})
        return out
    pol.act = recording_act
    return rec


def test_apex_vector_actor_end_to_end(gpu):
    from distributed_reinforcement_learning_b200.actor import ApexVectorActor
    from distributed_reinforcement_learning_b200.agent import apex
    from distributed_reinforcement_learning_b200.apex_learner import MAIN
    from distributed_reinforcement_learning_b200.apex_policy import NativeApexPolicy
    from distributed_reinforcement_learning_b200.distributed_queue import buffer_queue
    A, T, n, batch_size = 6, 5, 8, 16
    avail = [A if k % 2 else 4 for k in range(n)]
    agent = apex.Agent([84, 84, 4], A, 0.99, 40.0, "abs_one", 1e-4, 0.0, 1e14, "apex_e2e", "apex_e2e")
    agent.set_session(None)
    agent.target_to_main()
    q = buffer_queue.ApexFIFOQueue(T, [84, 84, 4], A, 256, batch_size, n)
    envs = [SyntheticEnv(k, episode_len=(7 if k % 2 else 12), life_loss=(3,) if k < 4 else ()) for k in range(n)]
    pol = NativeApexPolicy(n, num_action=A)
    rec = _recording(pol)
    np.random.seed(2025)
    va = ApexVectorActor(pol, envs, q, T, avail, learner=agent)
    memory = buffer_queue.Memory(capacity=1000)
    losses, buffer_step, finished = [], 0, []
    try:
        for unroll in range(5):           # host-parameter sync, then device to device from the learner
            finished += va.run_unroll()
            pushes = max(0, (unroll + 1) * T - 3 * T) - max(0, unroll * T - 3 * T)
            assert q.get_size() == pushes * n                  # the LocalBuffer gate, then one batch per step
            # the learner loop of train_apex.py:88-155: td error per batch -> Memory.add -> sample -> distributed_train
            while q.get_size():
                buffer_step += 1
                b = q.sample_batch(1)
                td = agent.get_td_error(state=b.state[0], next_state=b.next_state[0],
                                        previous_action=b.previous_action[0], action=b.action[0],
                                        reward=b.reward[0], done=b.done[0])
                for i in range(len(td)):
                    memory.add(td[i], [b.state[0][i], b.next_state[0][i], b.previous_action[0][i], b.action[0][i],
                                       b.reward[0][i], b.done[0][i]])
            if buffer_step > 10:
                minibatch, idxs, is_weight = memory.sample(batch_size)
                cols = list(zip(*minibatch))
                loss, td = agent.distributed_train(state=np.stack(cols[0]), next_state=np.stack(cols[1]),
                                                   previous_action=np.stack(cols[2]), action=np.stack(cols[3]),
                                                   reward=np.stack(cols[4]), done=np.stack(cols[5]),
                                                   is_weight=is_weight)
                for k, idx in enumerate(idxs):
                    memory.update(idx, td[k])
                losses.append(loss)
        assert len(losses) >= 2 and all(np.isfinite(x) for x in losses)
        for i, env in enumerate(envs):
            raw = [int(r["action"][i]) for r in rec]
            assert list(va.buffers[i].action) == raw
            assert env.actions == [a % avail[i] for a in raw]
            lost = [i < 4 and (t % env.episode_len) + 1 == 3 for t in range(len(rec))]
            assert list(va.buffers[i].done) == lost
            assert list(va.buffers[i].reward) == [-1 if l else r for l, r in zip(lost, env.rewards)]
        for r in rec:
            assert np.array_equal(r["q_action"], r["q"][np.arange(n), r["action"]])
        assert sorted((e["task"], e["episode"]) for e in finished) == sorted(
            (i, t // envs[i].episode_len) for i in range(n) for t in range(len(rec))
            if (t + 1) % envs[i].episode_len == 0)
        agent.sync_policy(pol)                                # device to device from the trained learner
        assert np.array_equal(pol.get_params(), agent._engine.get_params(MAIN))
    finally:
        pol.close()
        if agent._engine is not None:
            agent._engine.close()


class TrainingA3CQueue:
    """A3CFIFOQueue with the learner loop of train_a3c.py:85-110 behind it: every trajectory an actor appends is
    sampled and trained on at once (the reference's queue holds one unroll)."""

    def __init__(self, queue, agent):
        self.queue, self.agent, self.losses, self.batches = queue, agent, [], []

    def append_to_queue(self, **kw):
        self.queue.append_to_queue(**kw)
        batch = self.queue.sample_batch()
        self.batches.append(batch)
        self.losses.append(self.agent.train(state=batch.state[0], next_state=batch.next_state[0],
                                            previous_action=batch.previous_action[0], action=batch.action[0],
                                            reward=batch.reward[0], done=batch.done[0]))


def test_a3c_vector_actor_end_to_end(gpu):
    from distributed_reinforcement_learning_b200.actor import A3CVectorActor
    from distributed_reinforcement_learning_b200.agent import a3c
    from distributed_reinforcement_learning_b200.apex_policy import NativeA3CPolicy
    from distributed_reinforcement_learning_b200.distributed_queue import buffer_queue
    A, T, n = 6, 10, 8
    avail = [A if k % 2 else 4 for k in range(n)]
    agent = a3c.Agent([84, 84, 4], A, 0.99, 1e-4, 0.0, 1e9, 0.5, 0.01, 40.0, "abs_one", "a3c_e2e", "a3c_e2e")
    agent.set_session(None)
    q = TrainingA3CQueue(buffer_queue.A3CFIFOQueue(T, [84, 84, 4], A, n), agent)
    envs = [SyntheticEnv(10 + k, episode_len=(7 if k % 2 else 12), life_loss=(3,) if k < 4 else ()) for k in range(n)]
    pol = NativeA3CPolicy(n, num_action=A)
    rec = _recording(pol)
    np.random.seed(2026)
    va = A3CVectorActor(pol, envs, q, T, avail, learner=agent)
    finished = []
    try:
        for unroll in range(3):           # host-parameter sync, then device to device from the learner
            before = len(rec)
            finished += va.run_unroll()
            for i, env in enumerate(envs):
                b = q.batches[unroll * n + i]
                raw = [int(r["action"][i]) for r in rec[before:]]
                assert np.asarray(b.action[0]).tolist() == raw
                assert env.actions[before:] == [a % avail[i] for a in raw]
                for t in range(T):
                    step = before + t
                    lost = i < 4 and (step % env.episode_len) + 1 == 3
                    assert bool(b.done[0][t]) == lost
                    assert float(b.reward[0][t]) == (-1.0 if lost else env.rewards[step])
        for r in rec:
            assert np.array_equal(r["max_prob"], r["policy"][np.arange(n), r["action"]])
        assert len(q.losses) == 3 * n and all(np.isfinite(x).all() for x in q.losses)
        assert sorted((e["task"], e["episode"]) for e in finished) == sorted(
            (i, t // envs[i].episode_len) for i in range(n) for t in range(len(rec))
            if (t + 1) % envs[i].episode_len == 0)
        agent.sync_policy(pol)                                # device to device from the trained learner
        assert np.array_equal(pol.get_params(), agent._engine.get_params())
    finally:
        pol.close()
        if agent._engine is not None:
            agent._engine.close()
