"""The Ape-X replay memory on the GPU (NativeApexReplay, apex.Agent.device_memory / train_from_memory) against the host
memory (buffer_queue.Memory over drl_per_*) and the host learner loop of train_apex.py:82-155: tree parity through adds,
samples and updates (wrap, a leaf drawn twice, a leaf updated twice in one batch), storage after wrapping, ingest
priorities from the learner's |td|, the whole loop with and without CUDA graphs, the error paths, and a policy engine
acting and syncing beside the training thread."""
import random
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SHAPE = (84, 84, 4)


@pytest.fixture(scope="module")
def gpu(native):
    if native.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return native


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-300))) if a.size else 0.0


def _transitions(rng, n, A=4):
    return dict(state=rng.integers(0, 256, (n,) + SHAPE, dtype=np.uint8),
                next_state=rng.integers(0, 256, (n,) + SHAPE, dtype=np.uint8),
                previous_action=rng.integers(0, A, n).astype(np.int32), action=rng.integers(0, A, n).astype(np.int32),
                reward=(rng.standard_normal(n) * 2).astype(np.float32), done=rng.random(n) < 0.2)


def _fields(t):
    return (t["state"], t["next_state"], t["previous_action"], t["action"], t["reward"], t["done"])


def _agent(name, seed, graph):
    from distributed_reinforcement_learning_b200.agent import apex
    from distributed_reinforcement_learning_b200.model import apex_value
    a = apex.Agent(input_shape=SHAPE, num_action=4, discount_factor=0.99, gradient_clip_norm=40.0,
                   reward_clipping="abs_one", start_learning_rate=1e-3, end_learning_rate=0.0, learning_frame=1e6,
                   model_name=name, learner_name=name)
    a.use_cuda_graph = graph
    a._main = apex_value.init_params(seed, num_action=4, input_shape=SHAPE)
    a._target = apex_value.init_params(seed + 1, num_action=4, input_shape=SHAPE)
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


@pytest.mark.parametrize("capacity", [37, 256])
def test_tree_parity_with_host_memory(gpu, capacity):
    from distributed_reinforcement_learning_b200.apex_replay import NativeApexReplay
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import Memory
    rng = np.random.default_rng(capacity)
    rep, mem = NativeApexReplay(capacity), Memory(capacity)
    t = _transitions(rng, 1)
    one = {k: np.repeat(v, 40, axis=0) for k, v in t.items()}      # the stored records do not matter to the tree
    try:
        added, dup_draw, dup_update = 0, False, False
        for it in range(60):
            op = (1, 2, 0)[(it - 2) % 3] if it >= 2 else 0     # add, add, then sample / update / add
            if op == 0:
                n = int(rng.integers(1, 33))
                err = rng.exponential(1.0, n)
                if it == 30:
                    err[0] = 1e4                         # a dominant priority: its leaf is drawn several times
                rep.add(None, *[f[:n] for f in _fields(one)], error=err)
                for i in range(n):
                    mem.add(err[i], i)
                added += n
            elif op == 1:
                n = int(rng.choice([1, 5, 16, 32]))
                ti = _check_sample(rep, mem, n, rng.random(n))
                dup_draw |= len(set(ti.tolist())) < n
                last = ti
            else:
                idx = np.concatenate([last, last[:3]])                 # the same leaf twice in one batch
                err = rng.exponential(1.0, idx.size)
                rep.update(idx, err)
                for i in range(idx.size):
                    mem.update(int(idx[i]), float(err[i]))
                dup_update = True
            _check_tree(rep, mem)
        assert added > capacity and dup_draw and dup_update
    finally:
        rep.close()


def test_storage_after_wrap(gpu):
    from distributed_reinforcement_learning_b200.apex_replay import NativeApexReplay
    rng = np.random.default_rng(1)
    cap = 37
    rep = NativeApexReplay(cap)
    want = {}
    try:
        cursor = 0
        for n in (20, 20, 15, 9):
            t = _transitions(rng, n)
            rep.add(None, *_fields(t), error=rng.random(n))
            for i in range(n):
                want[(cursor + i) % cap] = {k: v[i] for k, v in t.items()}
            cursor = (cursor + n) % cap
        got = rep.read(0, cap)
        for row, w in want.items():
            for k in ("state", "next_state", "previous_action", "action", "reward"):
                assert np.array_equal(got[k][row], w[k]), (row, k)
            assert got["done"][row] == int(w["done"])
        assert rep.n_entries == cap
    finally:
        rep.close()


def test_ingest_priorities_from_the_learner(gpu):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import Memory
    rng = np.random.default_rng(2)
    agent = _agent("replay_ingest", 5, False)
    agent._get_engine(32)
    memory = agent.device_memory(256)
    mem = Memory(256)
    try:
        for n in (32, 40, 7):                             # 40: two chunks of the learner's batch
            t = _transitions(rng, n)
            memory.add(*_fields(t))
            td = agent.get_td_error(*_fields(t))
            for i in range(n):
                mem.add(td[i], i)
            _check_tree(memory.replay, mem)
        u = rng.random(32)
        _check_sample(memory.replay, mem, 32, u)
    finally:
        memory.close()


def _run_loop(agent, device, records, iters, seed, batch=32, capacity=256):
    """train_apex.py:82-155 (learner branch) for `iters` iterations; target_to_main every 5 train steps."""
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import Memory
    random.seed(seed)
    agent.target_to_main()
    memory = agent.device_memory(capacity) if device else Memory(capacity)
    out = dict(idx=[], loss=[], td=[])
    buffer_step = train_step = 0
    try:
        for it in range(iters):
            r = records[it % len(records)]
            buffer_step += 1
            if device:
                memory.add(*_fields(r))
            else:
                td_error = agent.get_td_error(*_fields(r))
                for i in range(len(td_error)):
                    memory.add(td_error[i], [r[k][i] for k in ("state", "next_state", "previous_action", "action",
                                                               "reward", "done")])
            if buffer_step > 2:
                train_step += 1
                if device:
                    loss, td_error = agent.train_from_memory(memory, batch)
                    idxs = memory.last_sample()[0].tolist()
                else:
                    minibatch, idxs, is_weight = memory.sample(batch)
                    minibatch = np.array(minibatch, dtype=object)
                    st = np.stack(minibatch[:, 0])
                    ns = np.stack(minibatch[:, 1])
                    pa = np.stack(minibatch[:, 2])
                    ac = np.stack(minibatch[:, 3])
                    rw = np.stack(minibatch[:, 4])
                    dn = np.stack(minibatch[:, 5])
                    loss, td_error = agent.distributed_train(state=st, next_state=ns, previous_action=pa, action=ac,
                                                             reward=rw, done=dn, is_weight=is_weight)
                    for i in range(len(idxs)):
                        memory.update(idxs[i], td_error[i])
                if train_step % 5 == 0:
                    agent.target_to_main()
                out["idx"].append(list(idxs))
                out["loss"].append(float(loss))
                out["td"].append(np.array(td_error, np.float64))
    finally:
        if device:
            memory.close()
    from distributed_reinforcement_learning_b200.apex_learner import MAIN, TARGET
    out["main"], out["target"] = agent._engine.get_params(MAIN), agent._engine.get_params(TARGET)
    return out


def _records(seed, n=6, T=32):
    rng = np.random.default_rng(seed)
    return [_transitions(rng, T) for _ in range(n)]


@pytest.mark.parametrize("graph", [False, True])
def test_loop_parity_host_vs_device(gpu, graph):
    records = _records(3)
    host = _run_loop(_agent("replay_host_%d" % graph, 11, graph), False, records, 22, seed=7)
    dev = _run_loop(_agent("replay_dev_%d" % graph, 11, graph), True, records, 22, seed=7)
    assert len(host["idx"]) == 20
    assert host["idx"] == dev["idx"]
    assert _rel(dev["loss"], host["loss"]) <= 1e-6, (dev["loss"], host["loss"])
    for a, b in zip(dev["td"], host["td"]):
        assert np.max(np.abs(a - b)) <= 1e-6 * max(1.0, np.max(np.abs(b)))
    for k in ("main", "target"):
        assert np.max(np.abs(dev[k] - host[k])) <= 1e-5 * np.max(np.abs(host[k])), k


def test_errors(gpu):
    from distributed_reinforcement_learning_b200 import _native as N
    from distributed_reinforcement_learning_b200.a3c_learner import NativeA3CLearner
    from distributed_reinforcement_learning_b200.apex_learner import NativeApexLearner
    from distributed_reinforcement_learning_b200.apex_replay import NativeApexReplay
    rng = np.random.default_rng(4)
    for cap in (1, 0, -5):
        with pytest.raises(N.DrlError, match="capacity"):
            NativeApexReplay(cap)
    rep = NativeApexReplay(64)
    eng = NativeApexLearner(batch=8, num_action=4)
    try:
        with pytest.raises(N.DrlError, match="empty") as ei:
            rep.sample(4, rng.random(4))
        assert ei.value.code == N.DRL_ERR_STATE
        with pytest.raises(N.DrlError, match="empty"):
            rep.step_async(eng, 0, rng.random(8))
        with pytest.raises(N.DrlError, match="exceeds the learner's batch"):
            rep.add(eng, *_fields(_transitions(rng, 9)))
        rep.add(eng, *_fields(_transitions(rng, 8)))
        with pytest.raises(N.DrlError, match="slot 5 out of range"):
            rep.step_async(eng, 5, rng.random(8))
        a3c = NativeA3CLearner(batch=8, num_action=4)
        try:
            with pytest.raises(N.DrlError, match="A3C"):
                rep.add(a3c, *_fields(_transitions(rng, 4)))
            with pytest.raises(N.DrlError, match="A3C"):
                rep.step_async(a3c, 0, rng.random(8))
        finally:
            a3c.close()
        if N.device_count() >= 2:
            other = NativeApexLearner(batch=8, num_action=4, device=1)
            try:
                with pytest.raises(N.DrlError, match="device"):
                    rep.step_async(other, 0, rng.random(8))
            finally:
                other.close()
        rep.step_async(eng, 1, rng.random(8))            # the memory still works after the refusals
        out, td = eng.wait()
        assert np.isfinite(out["loss"]) and td.shape == (8,)
    finally:
        eng.close()
        rep.close()


def test_train_from_memory_beside_a_policy_thread(gpu):
    from distributed_reinforcement_learning_b200.apex_policy import NativeApexPolicy
    records = _records(5, n=3)

    def run(with_actor):
        agent = _agent("replay_actor_%d" % with_actor, 21, True)
        random.seed(9)
        agent._get_engine(32)
        memory = agent.device_memory(128)
        stop, errors = threading.Event(), []
        pol = NativeApexPolicy(16, num_action=4)

        def actor():
            rng = np.random.default_rng(0)
            try:
                while not stop.is_set():
                    agent.sync_policy(pol)
                    pol.act(rng.integers(0, 256, (16,) + SHAPE, dtype=np.uint8), rng.integers(0, 4, 16),
                            epsilon=0.1)
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
                losses.append(agent.train_from_memory(memory, 32))
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
