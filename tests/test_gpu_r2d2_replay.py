"""The R2D2 sequence replay memory on the GPU (NativeR2D2Replay, r2d2.Agent.device_memory / train_from_memory) against
the host memory (buffer_queue.Memory over drl_per_*) and the host learner loop of train_r2d2.py:87-165: storage after
wrapping, the tree wiring (wrap, a leaf drawn twice, a leaf updated twice in one batch), ingest priorities from the
learner's batched |td| and their agreement with per-sequence get_td_error, the whole loop with and without CUDA graphs
at a small and at the reference configuration, the error paths, and a policy engine acting and syncing beside the
training thread."""
import random
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

A, L = 4, 64


@pytest.fixture(scope="module")
def gpu(native):
    if native.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return native


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-300))) if a.size else 0.0


def _sequences(rng, n, S, C=1):
    """One R2D2FIFOQueue.sample_batch() worth of sequences (h / c as the actors store them, [n, S, L])."""
    return dict(state=rng.integers(0, 256, (n, S, 84, 84, C), dtype=np.uint8),
                previous_action=rng.integers(0, A, (n, S)).astype(np.int32),
                action=rng.integers(0, A, (n, S)).astype(np.int32),
                h=(rng.standard_normal((n, S, L)) * 0.3).astype(np.float32),
                c=(rng.standard_normal((n, S, L)) * 0.3).astype(np.float32),
                reward=(rng.standard_normal((n, S)) * 2).astype(np.float32), done=rng.random((n, S)) < 0.1)


def _fields(t):
    """DeviceMemory.add's argument order."""
    return (t["state"], t["previous_action"], t["action"], t["h"], t["c"], t["reward"], t["done"])


def _rows(t):
    """NativeR2D2Replay.add's / NativeR2D2Learner.td_error's argument order (h0 / c0 at step 0)."""
    return (t["state"], t["previous_action"], t["action"], t["h"][:, 0], t["c"][:, 0], t["reward"], t["done"])


def _agent(name, seed, graph, S, burn_in, C=1):
    from distributed_reinforcement_learning_b200.agent import r2d2
    from distributed_reinforcement_learning_b200.model import r2d2_lstm
    a = r2d2.Agent(S, burn_in, [84, 84, C], A, L, 0.997, 1e-4, 1e-4, 1e9, 40.0, name, name)
    a.use_cuda_graph = graph
    kw = dict(num_action=A, lstm_size=L, input_shape=(84, 84, C))
    a._main = r2d2_lstm.init_params(seed, **kw)
    a._target = r2d2_lstm.init_params(seed + 1, **kw)
    z = np.zeros_like(a._main)
    a._opt = dict(m=z, v=z.copy(), step=0, beta1_power=0.9, beta2_power=0.999)
    return a


def _check_tree(rep, mem):
    assert rep.n_entries == mem.tree.n_entries
    assert _rel(rep.total(), mem.tree.total()) <= 1e-12, (rep.total(), mem.tree.total())
    assert _rel(rep.beta, mem.beta) <= 1e-12


def _check_sample(rep, mem, n, u):
    ti, di, pr, w = rep.sample(n, u)
    _, idxs, hw = mem.sample(n, u)
    assert ti.tolist() == idxs
    assert di.tolist() == [i - mem.capacity + 1 for i in idxs]
    assert _rel(pr, mem.last_priorities) <= 1e-12
    assert _rel(w, hw) <= 1e-12
    return ti


@pytest.mark.parametrize("C", [1, 4])
def test_storage_after_wrap(gpu, C):
    from distributed_reinforcement_learning_b200.r2d2_replay import NativeR2D2Replay
    rng = np.random.default_rng(C)
    cap, S = 37, 6
    rep = NativeR2D2Replay(cap, seq_len=S, num_action=A, input_shape=(84, 84, C))
    want = {}
    try:
        cursor = 0
        for n in (20, 20, 15, 9):
            t = _sequences(rng, n, S, C)
            rep.add(None, *_rows(t), error=rng.random(n))
            for i in range(n):
                want[(cursor + i) % cap] = {k: v[i] for k, v in t.items()}
            cursor = (cursor + n) % cap
        got = rep.read(0, cap)
        assert len(want) == cap
        for row, w in want.items():
            for k in ("state", "previous_action", "action", "reward"):
                assert np.array_equal(got[k][row], w[k]), (row, k)
            assert np.array_equal(got["done"][row], w["done"].astype(np.uint8)), row
            assert np.array_equal(got["h0"][row], w["h"][0]) and np.array_equal(got["c0"][row], w["c"][0]), row
        assert rep.n_entries == cap
    finally:
        rep.close()


def test_tree_wiring_against_host_memory(gpu):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import Memory
    from distributed_reinforcement_learning_b200.r2d2_replay import NativeR2D2Replay
    rng = np.random.default_rng(37)
    cap, S = 37, 2
    rep, mem = NativeR2D2Replay(cap, seq_len=S, num_action=A), Memory(cap)
    one = {k: np.repeat(v, 24, axis=0) for k, v in _sequences(rng, 1, S).items()}   # the records do not matter here
    try:
        dup_draw = False
        for it, n in enumerate((24, 20, 9)):             # 53 > 37: wraps
            err = rng.exponential(1.0, n)
            if it == 1:
                err[3] = 1e4                             # a dominant priority: its leaf is drawn several times
            rep.add(None, *[f[:n] for f in _rows(one)], error=err)
            for i in range(n):
                mem.add(err[i], i)
            _check_tree(rep, mem)
            ti = _check_sample(rep, mem, 16, rng.random(16))
            dup_draw |= len(set(ti.tolist())) < 16
            idx = np.concatenate([ti, ti[:3]])           # the same leaf twice in one batch
            e = rng.exponential(1.0, idx.size)
            rep.update(idx, e)
            for i in range(idx.size):
                mem.update(int(idx[i]), float(e[i]))
            _check_tree(rep, mem)
        assert dup_draw
    finally:
        rep.close()


def test_ingest_priorities_from_the_learner(gpu):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import Memory
    rng = np.random.default_rng(2)
    S, B = 6, 16
    agent = _agent("r2d2_replay_ingest", 5, False, S, 2)
    eng = agent._get_engine(B)
    memory = agent.device_memory(256)
    mem = Memory(256)
    try:
        for n in (16, 20, 3):                             # 20: two chunks of the learner's batch
            t = _sequences(rng, n, S)
            memory.add(*_fields(t))
            batched = np.concatenate([eng.td_error(*[f[lo:lo + B] for f in _rows(t)]) for lo in range(0, n, B)])
            for i in range(n):
                mem.add(batched[i], i)
            _check_tree(memory.replay, mem)
            # the reference's one-sequence-at-a-time priorities: the same to float32 rounding (another split-K order)
            single = np.array([agent.get_td_error(t["state"][i], t["previous_action"][i], t["action"][i], t["h"][i],
                                                  t["c"][i], t["reward"][i], t["done"][i]) for i in range(n)])
            assert np.max(np.abs(single - batched)) <= 1e-5 * np.max(np.abs(batched)), (single, batched)
        _check_sample(memory.replay, mem, 16, rng.random(16))
    finally:
        memory.close()


def _run_loop(agent, device, records, iters, seed, batch, capacity=256):
    """train_r2d2.py:87-165 (learner branch) for `iters` iterations of one queued batch each; main_to_target every 5
    train steps.  The host arm's priorities are the learner's batched |td| of each record, as the device ingest's."""
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import Memory
    random.seed(seed)
    agent.main_to_target()
    memory = agent.device_memory(capacity) if device else Memory(capacity)
    out = dict(idx=[], loss=[], td=[])
    buffer_step = train_step = 0
    try:
        for it in range(iters):
            r = records[it % len(records)]
            buffer_step += batch
            if device:
                memory.add(*_fields(r))
            else:
                td_error = agent._get_engine(batch).td_error(*_rows(r))
                for i in range(batch):
                    memory.add(td_error[i], [r["state"][i], r["previous_action"][i], r["action"][i], r["reward"][i],
                                             r["done"][i], r["h"][i], r["c"][i]])
            if buffer_step > batch * 2:
                train_step += 1
                if device:
                    loss, td_error = agent.train_from_memory(memory, batch)
                    idxs = memory.last_sample()[0].tolist()
                else:
                    minibatch, idxs, weight = memory.sample(batch)
                    cols = [[b[k] for b in minibatch] for k in range(7)]
                    loss, td_error = agent.train(state=cols[0], previous_action=cols[1], action=cols[2], h=cols[5],
                                                 c=cols[6], reward=cols[3], done=cols[4], weight=weight)
                    for i in range(len(idxs)):
                        memory.update(idxs[i], td_error[i])
                if train_step % 5 == 0:
                    agent.main_to_target()
                out["idx"].append(list(idxs))
                out["loss"].append(float(loss))
                out["td"].append(np.array(td_error, np.float64))
    finally:
        if device:
            memory.close()
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET
    out["main"], out["target"] = agent._engine.get_params(MAIN), agent._engine.get_params(TARGET)
    return out


@pytest.mark.parametrize("B,S,burn_in", [(4, 6, 2), (16, 15, 7)])
@pytest.mark.parametrize("graph", [False, True])
def test_loop_parity_host_vs_device(gpu, graph, B, S, burn_in):
    rng = np.random.default_rng(3)
    records = [_sequences(rng, B, S) for _ in range(6)]
    tag = "%d_%d_%d" % (graph, B, S)
    host = _run_loop(_agent("r2d2_replay_host_" + tag, 11, graph, S, burn_in), False, records, 22, 7, B)
    dev = _run_loop(_agent("r2d2_replay_dev_" + tag, 11, graph, S, burn_in), True, records, 22, 7, B)
    assert len(host["idx"]) == 20
    assert host["idx"] == dev["idx"]
    assert _rel(dev["loss"], host["loss"]) <= 1e-6, (dev["loss"], host["loss"])
    for a, b in zip(dev["td"], host["td"]):
        assert np.max(np.abs(a - b)) <= 1e-6 * max(1.0, np.max(np.abs(b)))
    for k in ("main", "target"):
        assert np.max(np.abs(dev[k] - host[k])) <= 1e-5 * np.max(np.abs(host[k])), k


def test_errors(gpu):
    import ctypes as C
    from distributed_reinforcement_learning_b200 import _native as N
    from distributed_reinforcement_learning_b200.r2d2_learner import NativeR2D2Learner
    from distributed_reinforcement_learning_b200.r2d2_replay import NativeR2D2Replay
    rng = np.random.default_rng(4)
    S = 6
    for cap in (1, 0, -5):
        with pytest.raises(N.DrlError, match="capacity"):
            NativeR2D2Replay(cap, seq_len=S)
    with pytest.raises(N.DrlError, match="seq_len"):
        NativeR2D2Replay(64, seq_len=1)
    rep = NativeR2D2Replay(64, seq_len=S, num_action=A)
    eng = NativeR2D2Learner(batch=8, seq_len=S, burn_in=2, num_action=A)
    try:
        with pytest.raises(N.DrlError, match="empty") as ei:
            rep.sample(4, rng.random(4))
        assert ei.value.code == N.DRL_ERR_STATE
        with pytest.raises(N.DrlError, match="empty"):
            rep.step_async(eng, 0, rng.random(8))
        with pytest.raises(N.DrlError, match="exceeds the learner's batch"):
            rep.add(eng, *_rows(_sequences(rng, 9, S)))
        for field, bad in (("action", A), ("previous_action", -1), ("action", -3), ("previous_action", A + 7)):
            t = _sequences(rng, 4, S)
            t[field][2, 3] = bad
            with pytest.raises(N.DrlError, match=r"sequence 2, step 3 is not in \[0, 4\)"):
                rep.add(eng, *_rows(t))
            with pytest.raises(N.DrlError, match=r"sequence 2, step 3 is not in \[0, 4\)"):
                rep.add(None, *_rows(t), error=rng.random(4))
        assert rep.n_entries == 0
        for kw in (dict(seq_len=S + 1), dict(input_shape=(84, 84, 4)), dict(num_action=A + 1)):
            args = dict(batch=8, seq_len=S, burn_in=2, num_action=A)
            args.update(kw)
            other = NativeR2D2Learner(**args)
            try:
                with pytest.raises(N.DrlError, match="the learner has seq_len"):
                    rep.add(other, *_rows(_sequences(rng, 2, S)))
                with pytest.raises(N.DrlError, match="the learner has seq_len"):
                    rep.step_async(other, 0, rng.random(8))
            finally:
                other.close()
        if N.device_count() >= 2:
            other = NativeR2D2Learner(batch=8, seq_len=S, burn_in=2, num_action=A, device=1)
            try:
                with pytest.raises(N.DrlError, match="device"):
                    rep.step_async(other, 0, rng.random(8))
            finally:
                other.close()
        rep.add(eng, *_rows(_sequences(rng, 8, S)))
        with pytest.raises(N.DrlError, match="slot 5 out of range"):
            rep.step_async(eng, 5, rng.random(8))
        for bad in (1.5, -0.25, float("nan")):
            u = rng.random(8)
            u[6] = bad
            with pytest.raises(N.DrlError, match=r"is not in \[0, 1\]"):
                rep.step_async(eng, 0, u)
            with pytest.raises(N.DrlError, match=r"is not in \[0, 1\]"):
                rep.sample(8, u)
        u = np.zeros(8)
        h = rep._h
        assert N.lib.drl_r2d2_replay_add(h, eng._h, 2, *[None] * 7, None) == N.DRL_ERR_INVALID
        assert "null input pointer" in N.lib.drl_last_error().decode()
        assert N.lib.drl_r2d2_replay_step_async(h, eng._h, 0, None) == N.DRL_ERR_INVALID
        assert N.lib.drl_r2d2_replay_step_async(h, None, 0, N.ptr(u)) == N.DRL_ERR_INVALID
        assert "null r2d2 handle" in N.lib.drl_last_error().decode()
        assert N.lib.drl_r2d2_replay_sample(h, 4, None, N.ptr(u), N.ptr(u), N.ptr(u), N.ptr(u)) == N.DRL_ERR_INVALID
        assert N.lib.drl_r2d2_replay_update(h, 2, None, N.ptr(u)) == N.DRL_ERR_INVALID
        assert N.lib.drl_r2d2_replay_total(h, None) == N.DRL_ERR_INVALID
        assert N.lib.drl_r2d2_replay_size(h, None) == N.DRL_ERR_INVALID
        assert N.lib.drl_r2d2_replay_beta(h, None) == N.DRL_ERR_INVALID
        with pytest.raises(N.DrlError, match="not a leaf index"):
            rep.update([5], [1.0])
        with pytest.raises(N.DrlError, match="not inside"):
            rep.read(60, 5)
        n_entries, beta = C.c_int64(), C.c_double()
        assert N.lib.drl_r2d2_replay_size(h, C.byref(n_entries)) == N.DRL_OK and n_entries.value == 8
        assert N.lib.drl_r2d2_replay_beta(h, C.byref(beta)) == N.DRL_OK
        rep.step_async(eng, 1, rng.random(8))            # the memory still works after the refusals
        out, td = eng.wait()
        assert np.isfinite(out["loss"]) and td.shape == (8,) and np.all(np.isfinite(td))
    finally:
        eng.close()
        rep.close()


def test_train_from_memory_beside_a_policy_thread(gpu):
    from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
    S, B = 6, 8
    rng = np.random.default_rng(5)
    records = [_sequences(rng, B, S) for _ in range(3)]

    def run(with_actor):
        agent = _agent("r2d2_replay_actor_%d" % with_actor, 21, True, S, 2)
        random.seed(9)
        agent._get_engine(B)
        memory = agent.device_memory(64)
        stop, errors = threading.Event(), []
        pol = NativeR2D2Policy(16, num_action=A)

        def actor():
            r = np.random.default_rng(0)
            try:
                while not stop.is_set():
                    agent.sync_policy(pol)
                    pol.act(r.integers(0, 256, (16, 84, 84, 1), dtype=np.uint8), r.integers(0, A, 16),
                            r.standard_normal((16, L)).astype(np.float32),
                            r.standard_normal((16, L)).astype(np.float32), epsilon=0.1)
            except Exception as e:                      # pragma: no cover
                errors.append(e)

        th = threading.Thread(target=actor) if with_actor else None
        losses = []
        try:
            for r in records:
                memory.add(*_fields(r))
            if th:
                th.start()
            for _ in range(10):
                losses.append(agent.train_from_memory(memory, B))
        finally:
            stop.set()
            if th:
                th.join()
            pol.close()
            memory.close()
        assert not errors, errors
        return [(float(l), np.asarray(t).copy()) for l, t in losses]

    a, b = run(False), run(True)
    for (la, ta), (lb, tb) in zip(a, b):
        assert la == lb and np.array_equal(ta, tb)
