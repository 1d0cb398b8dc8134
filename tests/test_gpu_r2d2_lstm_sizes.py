"""GPU tests of the R2D2 learner and its device replay memory at lstm_size 256 and 512, where the LSTM recurrence runs on
a thread-block cluster (csrc/r2d2_cluster.cuh): full-step parity with the float64 oracle at 1e-4 relative, the two
recurrence kernels against float64 fed from the step's own buffers, bitwise determinism, td_error / act, the agent
surface, the device replay loop against the host Memory, and what stays rejected."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

import r2d2_lstm_parity as lp
from oracle import r2d2_torch as rt

pytestmark = pytest.mark.gpu

SIZES = [256, 512]


def _check(errs):
    bad = lp.r2d2_failures(errs)
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:10]


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("C_", [1, 4])
@pytest.mark.parametrize("L", SIZES)
def test_step_parity_small(native, L, C_, mode, graph):
    """B = 3 (2 with four channels), S = 6: a done at t = 0, mid-sequence and t = S - 1 of every sequence; two steps."""
    _check(lp.compare_step(3 if C_ == 1 else 2, 6, 2, C=C_, L=L, steps=2, math_mode=mode, use_cuda_graph=graph))


def test_step_parity_benchmark_shape(native):
    """The benchmarked R2D2 shape: B = 16, S = 80, burn-in 40, 84x84x1, A = 4, at L = 512 (two clusters of 16 CTAs
    and more than one R-sequence chunk each)."""
    _check(lp.compare_step(16, 80, 40, L=512, use_cuda_graph=True, done_ends=False))


@pytest.mark.parametrize("L,B,S,bi", [(256, 3, 6, 2), (256, 9, 12, 4), (512, 3, 6, 2), (512, 16, 80, 40)])
def test_recurrence_kernels_against_own_buffers(native, L, B, S, bi):
    A, C_ = 4, 1
    ref, eng = lp.setup(B, S, bi, A, C_, L)
    try:
        b = lp.make_batch(B, S, A, C_, L, 11, done_ends=True)
        eng.stage(0, b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"], b["done"],
                  b["weight"])
        eng.step(0)
        buf = lp.read_recurrence(eng, B, S, L)
        # the step read the parameters before its update: the oracle's untrained copy
        W = ref.params["lstm.w"].detach().double().numpy()
        Wh, bias = W[W.shape[0] - L:], ref.params["lstm.b"].detach().double().numpy()
        # the state entering step 0 is the staged (h0, c0)
        assert np.array_equal(buf["hin"][0], b["h"][:, 0].astype(np.float64))
        assert np.array_equal(buf["cin"][0], b["c"][:, 0].astype(np.float64))
        fwd = lp.forward_check(buf, bias, Wh, b["done"], L)
        assert all(v <= 1.0 for v in fwd.values()), fwd
        err = lp.backward_error(buf, Wh, b["done"], L)
        assert err <= 2e-5, err
    finally:
        eng.close()


def _staged(L, B=4, S=10, bi=3, seed=5, **kw):
    ref, eng = lp.setup(B, S, bi, 4, 1, L, **kw)
    b = lp.make_batch(B, S, 4, 1, L, seed, done_ends=True)
    for slot in range(eng.num_slots):
        eng.stage(slot, b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"],
                  b["done"], b["weight"])
    return eng


def _state(eng, out, td):
    return [np.float32(out["loss"]), np.float32(out["grad_norm"]), td, eng.get_grads(), eng.get_params(),
            eng.get_opt_state()["m"], eng.get_opt_state()["v"], eng.read_buffer("dz", eng.B * eng.S * 4 * eng.L)]


def _bit_equal(x, y):
    return all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(x, y))


@pytest.mark.parametrize("L", SIZES)
def test_determinism(native, L):
    """Two learners agree bit for bit over two steps; a graph learner equals an eager one; forward_backward + apply
    equals step."""
    runs = []
    for kw in (dict(use_cuda_graph=False), dict(use_cuda_graph=False), dict(use_cuda_graph=True)):
        eng = _staged(L, **kw)
        try:
            runs.append([_state(eng, *eng.step(s)) for s in range(2)])
        finally:
            eng.close()
    assert _bit_equal(runs[0][0], runs[1][0]) and _bit_equal(runs[0][1], runs[1][1])
    assert _bit_equal(runs[0][0], runs[2][0]) and _bit_equal(runs[0][1], runs[2][1])
    eng = _staged(L)
    try:
        got = []
        for s in range(2):
            native.check(eng._fn("forward_backward")(eng._h, s))
            native.check(eng._fn("apply")(eng._h, C.c_float(1.0)))
            got.append(_state(eng, *eng.wait()))
        assert _bit_equal(got[0], runs[0][0]) and _bit_equal(got[1], runs[0][1])
    finally:
        eng.close()


@pytest.mark.parametrize("L", SIZES)
def test_td_error_and_act(native, L):
    A, S, bi, B = 4, 8, 3, 4
    ref, eng = lp.setup(B, S, bi, A, 1, L)
    try:
        for n in (1, B):
            b = lp.make_batch(n, S, A, 1, L, 77 + n, done_ends=True)
            rows = [b[k] for k in rt.TRAIN_FIELDS[:-1]]
            td = eng.td_error(b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"],
                              b["done"])
            exp = np.asarray([ref.get_td_error(*[r[i] for r in rows]) for i in range(n)])
            t = eng.taps(n)
            o = ref.losses(*rows)
            # |td| = |mean_t(target - q)| cancels: each sequence's error is judged against the size of the terms it
            # averages, mean_t |target - q|, when that is larger than |td| itself
            diff = (o["target_value"] - o["state_action_value"]).detach().numpy()
            scale = np.maximum(np.abs(exp), np.mean(np.abs(diff), axis=1))
            assert np.max(np.abs(td - exp) / scale) < lp.TOL, n
            for k in ("main_q", "target_q", "target_value", "state_action_value"):
                assert lp.rel_err(t[k], o[k].detach().numpy()) < lp.TOL, (n, k)
        for n in (1, B * S):
            b = lp.make_batch(n, 2, A, 1, L, 91 + n)
            q, h2, c2 = eng.act(b["state"][:, 0], b["previous_action"][:, 0], b["h"][:, 0], b["c"][:, 0])
            rq, rh, rc = ref.step_q(b["state"][:, 0], b["h"][:, 0], b["c"][:, 0], b["previous_action"][:, 0])
            assert h2.shape == (n, L) and c2.shape == (n, L)
            for got, exp in ((q, rq), (h2, rh), (c2, rc)):
                assert lp.rel_err(got, exp) < lp.TOL, n
    finally:
        eng.close()


def _agent(name, L, S=6, bi=2, seed=3, graph=False):
    from distributed_reinforcement_learning_b200.agent import r2d2
    from distributed_reinforcement_learning_b200.model import r2d2_lstm
    a = r2d2.Agent(S, bi, [84, 84, 1], 4, L, 0.997, 1e-4, 1e-4, 1e9, 40.0, name, name)
    a.use_cuda_graph = graph
    kw = dict(num_action=4, lstm_size=L, input_shape=(84, 84, 1))
    a._main = r2d2_lstm.init_params(seed, **kw)
    a._target = r2d2_lstm.init_params(seed + 1, **kw)
    z = np.zeros_like(a._main)
    a._opt = dict(m=z, v=z.copy(), step=0, beta1_power=0.9, beta2_power=0.999)
    return a


def test_agent_at_512(native, tmp_path):
    L, S = 512, 6
    a = _agent("r2d2_lstm512_agent", L, S)
    q = rt.make_sequences(4, S=S, L=L, seed=5)
    td = a.get_td_error(q["state"][0], q["previous_action"][0], q["action"][0], q["h"][0], q["c"][0], q["reward"][0],
                        q["done"][0])
    assert np.isfinite(td) and td >= 0
    a.main_to_target()
    for _ in range(2):
        loss, tde = a.train(list(q["state"]), list(q["previous_action"]), list(q["action"]), list(q["h"]), list(q["c"]),
                            list(q["reward"]), list(q["done"]), np.ones(4, np.float32))
        assert np.isfinite(loss) and tde.shape == (4,)
    action, qa, h2, c2 = a.get_action(q["state"][0][0], q["h"][0][0], q["c"][0][0], 0, epsilon=0.0)
    assert h2.shape == (L,) and c2.shape == (L,) and np.isfinite(qa) and 0 <= action < 4
    path = str(tmp_path / "r2d2_512")
    a.save_weights(path)
    b = _agent("r2d2_lstm512_agent_b", L, S, seed=9)
    b.load_weights(path)
    b._get_engine(4)
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET
    for w in (MAIN, TARGET):
        assert np.array_equal(a._engine.get_params(w), b._engine.get_params(w))
    assert b._engine.get_opt_state()["step"] == 2
    assert np.array_equal(a._engine.get_opt_state()["m"], b._engine.get_opt_state()["m"])
    small = _agent("r2d2_lstm64_agent", 64, S)
    with pytest.raises(ValueError, match="lstm_size"):
        small.load_weights(path)


def _run_loop(agent, device, records, iters, seed, batch, capacity=64):
    """tests/test_gpu_r2d2_replay.py's learner loop: host Memory or DeviceMemory, the learner's |td| as priorities."""
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import Memory
    random.seed(seed)
    agent.main_to_target()
    memory = agent.device_memory(capacity) if device else Memory(capacity)
    out = dict(idx=[], loss=[])
    step = 0
    try:
        for it in range(iters):
            r = records[it % len(records)]
            if device:
                memory.add(r["state"], r["previous_action"], r["action"], r["h"], r["c"], r["reward"], r["done"])
            else:
                td = agent._get_engine(batch).td_error(r["state"], r["previous_action"], r["action"], r["h"][:, 0],
                                                       r["c"][:, 0], r["reward"], r["done"])
                for i in range(batch):
                    memory.add(td[i], [r["state"][i], r["previous_action"][i], r["action"][i], r["reward"][i],
                                       r["done"][i], r["h"][i], r["c"][i]])
            if it >= 2:
                step += 1
                if device:
                    loss, td = agent.train_from_memory(memory, batch)
                    idxs = memory.last_sample()[0].tolist()
                else:
                    minibatch, idxs, weight = memory.sample(batch)
                    cols = [[b[k] for b in minibatch] for k in range(7)]
                    loss, td = agent.train(state=cols[0], previous_action=cols[1], action=cols[2], h=cols[5], c=cols[6],
                                           reward=cols[3], done=cols[4], weight=weight)
                    for i in range(len(idxs)):
                        memory.update(idxs[i], td[i])
                out["idx"].append(list(idxs))
                out["loss"].append(float(loss))
    finally:
        if device:
            memory.close()
    return out


def _device_replay_samples_the_host_memory(L):
    """The device replay memory at width L samples the same indices as the host Memory and gives identical losses."""
    S, bi, B = 6, 2, 4
    rng = np.random.default_rng(3)
    records = []
    for _ in range(4):
        q = rt.make_sequences(B, S=S, L=L, seed=int(rng.integers(1 << 30)))
        q["h"] = np.repeat(q["h"][:, :1], S, 1)
        q["c"] = np.repeat(q["c"][:, :1], S, 1)
        records.append(q)
    host = _run_loop(_agent("r2d2_lstm%d_host" % L, L, S, bi), False, records, 10, 7, B)
    dev = _run_loop(_agent("r2d2_lstm%d_dev" % L, L, S, bi), True, records, 10, 7, B)
    assert len(host["idx"]) == 8 and host["idx"] == dev["idx"]
    assert host["loss"] == dev["loss"]


def test_device_replay_at_512_samples_the_host_memory(native):
    _device_replay_samples_the_host_memory(512)


def test_device_replay_at_256_samples_the_host_memory(native):
    _device_replay_samples_the_host_memory(256)


def test_replay_storage_and_width_checks(native):
    from distributed_reinforcement_learning_b200.r2d2_learner import NativeR2D2Learner
    from distributed_reinforcement_learning_b200.r2d2_replay import NativeR2D2Replay
    L, S = 512, 6
    rep = NativeR2D2Replay(8, seq_len=S, lstm_size=L)
    eng = NativeR2D2Learner(batch=2, seq_len=S, burn_in=2, lstm_size=L)
    eng64 = NativeR2D2Learner(batch=2, seq_len=S, burn_in=2)
    try:
        q = rt.make_sequences(2, S=S, L=L, seed=1)
        rep.add(eng, q["state"], q["previous_action"], q["action"], q["h"][:, 0], q["c"][:, 0], q["reward"], q["done"])
        r = rep.read(0, 2)
        assert np.array_equal(r["h0"], q["h"][:, 0]) and np.array_equal(r["c0"], q["c"][:, 0])
        with pytest.raises(ValueError):
            rep.add(None, q["state"], q["previous_action"], q["action"], q["h"][:, 0, :64], q["c"][:, 0, :64],
                    q["reward"], q["done"], error=np.ones(2))
        with pytest.raises(native.DrlError, match="lstm_size"):
            rep.add(eng64, q["state"], q["previous_action"], q["action"], q["h"][:, 0], q["c"][:, 0], q["reward"],
                    q["done"])
        with pytest.raises(native.DrlError, match="lstm_size"):
            rep.step_async(eng64, 0, np.full(2, 0.5))
    finally:
        for x in (rep, eng, eng64):
            x.close()


def test_add_from_queue_rejects_a_width_mismatch(native):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import R2D2DeviceFIFOQueue
    from distributed_reinforcement_learning_b200.r2d2_learner import NativeR2D2Learner
    from distributed_reinforcement_learning_b200.r2d2_replay import NativeR2D2Replay
    S = 6
    queue = R2D2DeviceFIFOQueue(S, (84, 84, 1), 4, 4, 2, 1, 64)
    rep = NativeR2D2Replay(8, seq_len=S, lstm_size=512)
    eng = NativeR2D2Learner(batch=2, seq_len=S, burn_in=2, lstm_size=512)
    try:
        with pytest.raises(native.DrlError, match="lstm_size"):
            rep.add_from_queue(eng, queue, timeout_ms=0)
    finally:
        for x in (rep, eng, queue):
            x.close()


def test_rejections(native):
    from distributed_reinforcement_learning_b200.r2d2_learner import NativeR2D2Learner
    from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
    from distributed_reinforcement_learning_b200.r2d2_replay import NativeR2D2Replay
    for L in (32, 100, 128, 1024):
        with pytest.raises(native.DrlError, match="lstm_size") as ei:
            NativeR2D2Learner(batch=2, lstm_size=L)
        assert ei.value.code == native.DRL_ERR_INVALID and "256" in str(ei.value) and "512" in str(ei.value)
        with pytest.raises(native.DrlError, match="lstm_size"):
            NativeR2D2Replay(8, lstm_size=L)
    eng = NativeR2D2Learner(batch=2, seq_len=6, burn_in=2, lstm_size=512)
    pol = NativeR2D2Policy(4)
    try:
        size, fwd, bwd = eng.recurrence_clusters()
        assert size == 16 and fwd >= 1 and bwd >= 1
        with pytest.raises(native.DrlError, match="lstm_size") as ei:
            pol.sync_from(eng)
        assert ei.value.code == native.DRL_ERR_INVALID
    finally:
        pol.close()
        eng.close()


def test_actors_reject_a_wide_agent(native):
    from distributed_reinforcement_learning_b200.actor import R2D2VectorActor
    from distributed_reinforcement_learning_b200.actor_server import R2D2PolicyServer
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import R2D2DeviceFIFOQueue
    from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
    agent = _agent("r2d2_lstm512_actor", 512)
    pol = NativeR2D2Policy(2)
    queue = R2D2DeviceFIFOQueue(6, (84, 84, 1), 4, 4, 2, 1, 64)

    class Env:
        def reset(self):
            return np.zeros((84, 84, 1), np.uint8)

    try:
        with pytest.raises(ValueError, match="lstm_size"):
            R2D2VectorActor(pol, [Env()], queue, 6, learner=agent)
        with pytest.raises(ValueError, match="lstm_size"):
            R2D2PolicyServer(pol, queue, object(), learner=agent)
    finally:
        pol.close()
        queue.close()
