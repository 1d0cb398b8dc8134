"""GPU tests of the R2D2 learner's n-step double-Q targets and mixed max / mean priorities (DESIGN.md section 22): full
steps against the float64 oracle at 1e-4 over widths, horizons, priority rules, math modes, graph / eager and three
consecutive steps; r2d2_td_nstep_kernel against float64 fed from the step's own q buffers; n = 1 against a learner built
without the new arguments; bitwise determinism; the device replay memory under the mixed rule against the host Memory;
and the Agent setters keeping the learner's state."""
import ctypes as C

import numpy as np
import pytest
import torch

import r2d2_nstep_oracle as no
from oracle import r2d2_torch as rt

pytestmark = pytest.mark.gpu

GAMMA32 = float(np.float32(rt.DEFAULT_CFG["discount_factor"]))


def _check(errs):
    bad = no.r2d2_failures(errs)
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:10]


# S = 10, burn-in 2: Nt = 7, so n = 7 is n = Nt.  Every (L, n) pair runs; eta, the math mode and graph / eager alternate
# so each value of each meets every width.
GRID = [(64, 3, None, 1, False), (64, 5, 0.9, 2, True), (64, 7, 0.9, 1, True),
        (256, 3, 0.9, 2, False), (256, 5, None, 1, True), (256, 7, None, 2, False),
        (512, 3, None, 2, True), (512, 5, 0.9, 1, False), (512, 7, 0.9, 2, True)]


@pytest.mark.parametrize("L,n,eta,mode,graph", GRID)
def test_step_parity(native, L, n, eta, mode, graph):
    """B = 3, S = 10, burn-in 2, dones at rate 0.3 (inside the horizons), three consecutive steps."""
    _check(no.compare_step(3, 10, 2, n, eta, L=L, steps=3, math_mode=mode, use_cuda_graph=graph))


def test_step_parity_benchmark_shape(native):
    """The benchmarked R2D2 shape, B = 16, S = 80, burn-in 40, at L = 512 with n = 5 and eta = 0.9, three steps."""
    _check(no.compare_step(16, 80, 40, 5, 0.9, L=512, steps=3, done_rate=0.02, use_cuda_graph=True))


def _bound_failures(name, got, ref, bound, Nt):
    """(sequence, window) of every element of a [B, Nt] (or [B]) output outside its bound."""
    got, ref, bound = (np.asarray(x, np.float64) for x in (got, ref, bound))
    bad = np.argwhere(np.abs(got - ref) > bound + 1e-300)
    return ["%s: sequence %d%s got %r want %r (bound %.3g)" % (name, i[0], ", window %d" % i[1] if len(i) > 1 else "",
                                                               got[tuple(i)], ref[tuple(i)], bound[tuple(i)])
            for i in bad[:8]]


@pytest.mark.parametrize("L,n,eta", [(64, 5, 0.9), (64, 7, None), (512, 3, 0.9), (256, 1, 0.9)])
def test_td_kernel_against_its_own_q_buffers(native, L, n, eta):
    B, S, bi, A = 5, 10, 2, 4
    Nt = S - bi - 1
    k = dict(num_action=A, lstm_size=L, input_shape=(84, 84, 1))
    eng = no.native(B, S, bi, A, 1, L, rt.init_params(0, torch.float32, **k), rt.init_params(1, torch.float32, **k),
                    n_step=n, priority_eta=eta)
    try:
        b = no.make_batch(B, S, A, 1, L, 321)
        eng.stage(0, b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"], b["done"],
                  b["weight"])
        out, td = eng.step(0)
        taps = eng.taps()
        dq = eng.read_buffer("dq", B * S * 32).reshape(B * S, 32)
        dmean = eng.read_buffer("dmean", B * S * 32).reshape(B * S, 32)
    finally:
        eng.close()
    ref = no.td_reference(taps["main_q"], taps["target_q"], b, bi, GAMMA32, B, S, A, n, eta)
    got = dict(target_value=taps["target_value"], sav=taps["state_action_value"], td=td)
    msgs = []
    for key in ("target_value", "sav", "td"):
        msgs += _bound_failures(key, got[key], ref[key], ref["bound/" + key], Nt)
    assert abs(out["loss"] - ref["loss"]) <= ref["bound/loss"], (out["loss"], ref["loss"])
    t = np.arange(B * S) // B
    rows = (t >= bi) & (t < S - 1)
    assert np.all(np.abs(dq[:, :A] - ref["dq"]) <= ref["bound/dq"] + 1e-300)
    assert np.all(np.abs(dmean[:, 0] - ref["dmean"]) <= ref["bound/dmean"] + 1e-300)
    assert not np.any(dq[~rows]) and not np.any(dq[:, A:]) and not np.any(dmean[:, 1:])
    assert not msgs, msgs


def _staged(L=64, B=4, S=10, bi=2, seed=5, **kw):
    k = dict(num_action=4, lstm_size=L, input_shape=(84, 84, 1))
    eng = no.native(B, S, bi, 4, 1, L, rt.init_params(0, torch.float32, **k), rt.init_params(1, torch.float32, **k),
                    **kw)
    for s in range(eng.num_slots):
        b = no.make_batch(B, S, 4, 1, L, seed + s)
        eng.stage(s, b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"], b["done"],
                  b["weight"])
    return eng


def _state(eng, out, td):
    return dict(loss=np.float32(out["loss"]), td=td.copy(), params=eng.get_params(), m=eng.get_opt_state()["m"])


def _run(steps=2, **kw):
    eng = _staged(**kw)
    try:
        return [_state(eng, *eng.step(s)) for s in range(steps)]
    finally:
        eng.close()


def _equal(a, b, keys=("loss", "td", "params", "m")):
    return all(np.array_equal(x[k], y[k]) for x, y in zip(a, b) for k in keys)


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("L", [64, 512])
def test_n1_is_the_reference_learner(native, L, graph):
    """n = 1 with eta None is bit for bit the learner built without the new arguments; with eta = 0.9 the losses and
    parameters stay bit-equal and |td| is the mixed rule of the same windows."""
    base = _run(L=L, use_cuda_graph=graph)
    assert _equal(_run(L=L, use_cuda_graph=graph, n_step=1, priority_eta=None), base)
    mixed = _run(L=L, use_cuda_graph=graph, n_step=1, priority_eta=0.9)
    assert _equal(mixed, base, ("loss", "params", "m"))
    eng = _staged(L=L, use_cuda_graph=graph, n_step=1, priority_eta=0.9)
    try:
        _, td = eng.step(0)
        t = eng.taps()
    finally:
        eng.close()
    diff = t["target_value"].astype(np.float64) - t["state_action_value"]
    assert np.max(np.abs(td - no.priority(diff, 0.9))) <= 1e-6 * np.max(td)
    assert not np.array_equal(td, base[0]["td"])


@pytest.mark.parametrize("L", [64, 256])
def test_determinism(native, L):
    """Repeated, graph and eager learners agree bit for bit over two steps; forward_backward + apply equals step."""
    kw = dict(L=L, n_step=5, priority_eta=0.9)
    first = _run(use_cuda_graph=False, **kw)
    assert _equal(_run(use_cuda_graph=False, **kw), first)
    assert _equal(_run(use_cuda_graph=True, **kw), first)
    eng = _staged(**kw)
    try:
        got = []
        for s in range(2):
            native.check(eng._fn("forward_backward")(eng._h, s))
            native.check(eng._fn("apply")(eng._h, C.c_float(1.0)))
            got.append(_state(eng, *eng.wait()))
    finally:
        eng.close()
    assert _equal(got, first)


def test_device_replay_with_the_mixed_rule_equals_the_host_memory(native):
    """DeviceMemory.add stores the learner's batched mixed-rule |td| as the host Memory does; the loop samples the same
    indices, with the same losses and |td|, as the host loop (tests/test_gpu_r2d2_replay.py's loop)."""
    import test_gpu_r2d2_replay as tr
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import Memory
    rng = np.random.default_rng(2)
    S, B = 15, 16
    agent = tr._agent("r2d2_nstep_ingest", 5, False, S, 7)
    agent.set_n_step(5)
    agent.set_priority_eta(0.9)
    eng = agent._get_engine(B)
    assert (eng.n_step, eng.priority_eta) == (5, 0.9)
    memory = agent.device_memory(256)
    mem = Memory(256)
    try:
        for n in (16, 20):
            t = tr._sequences(rng, n, S)
            memory.add(*tr._fields(t))
            batched = np.concatenate([eng.td_error(*[f[lo:lo + B] for f in tr._rows(t)]) for lo in range(0, n, B)])
            for i in range(n):
                mem.add(batched[i], i)
            tr._check_tree(memory.replay, mem)
        tr._check_sample(memory.replay, mem, 16, rng.random(16))
    finally:
        memory.close()
    records = [tr._sequences(rng, 4, 6) for _ in range(6)]
    arms = []
    for device in (False, True):
        a = tr._agent("r2d2_nstep_loop_%d" % device, 11, True, 6, 2)
        a.set_n_step(3)
        a.set_priority_eta(0.9)
        arms.append(tr._run_loop(a, device, records, 12, 7, 4))
    host, dev = arms
    assert host["idx"] == dev["idx"]
    assert tr._rel(dev["loss"], host["loss"]) <= 1e-6
    for a, b in zip(dev["td"], host["td"]):
        assert np.max(np.abs(a - b)) <= 1e-6 * max(1.0, np.max(np.abs(b)))


@pytest.mark.parametrize("graph", [True, False])
def test_add_from_queue_with_the_mixed_rule_is_bitwise_add(native, graph):
    import test_gpu_r2d2_queue as tq
    params = tq._params()
    hq, dq, _ = tq._arms(16, unrolls=2, params=params)
    agents = [tq._agent(params, "rq_nstep_%s_%d" % (k, graph), graph) for k in ("host", "dev")]
    for a in agents:
        a.set_n_step(5)
        a.set_priority_eta(0.9)
    mem_h, mem_d = agents[0].device_memory(64), agents[1].device_memory(64)
    try:
        for _ in range(2):
            b = hq.sample_batch()
            mem_h.add(b.state, b.previous_action, b.action, b.previous_h, b.previous_c, b.reward, b.done)
            mem_d.add_from_queue(dq)
        assert mem_h.n_entries == mem_d.n_entries == 32
        assert mem_h.total() == mem_d.total()
        rh, rd = mem_h.replay.read(0, 32), mem_d.replay.read(0, 32)
        for k in rh:
            assert np.array_equal(rh[k], rd[k]), k
        u = np.random.RandomState(5).random_sample(tq.B)
        for x, y in zip(mem_h.replay.sample(tq.B, u), mem_d.replay.sample(tq.B, u)):
            assert np.array_equal(x, y)
    finally:
        mem_h.close()
        mem_d.close()


def test_agent_switch_keeps_parameters_and_adam_state(native):
    from distributed_reinforcement_learning_b200.agent import r2d2
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET
    S, bi = 10, 2
    a = r2d2.Agent(S, bi, [84, 84, 1], 4, 64, 0.997, 1e-4, 1e-4, 1e9, 40.0, "r2d2_nstep_switch", "r2d2_nstep_switch")
    q = rt.make_sequences(4, S=S, seed=5)
    args = (list(q["state"]), list(q["previous_action"]), list(q["action"]), list(q["h"]), list(q["c"]),
            list(q["reward"]), list(q["done"]), np.ones(4, np.float32))
    a.train(*args)
    before = a._engine
    keep = (before.get_params(MAIN), before.get_params(TARGET), before.get_opt_state())
    a.set_n_step(5)
    a.set_priority_eta(0.9)
    assert a._engine is None
    eng = a._get_engine(4)
    assert (eng.n_step, eng.priority_eta) == (5, 0.9)
    st = eng.get_opt_state()
    assert np.array_equal(eng.get_params(MAIN), keep[0]) and np.array_equal(eng.get_params(TARGET), keep[1])
    assert st["step"] == keep[2]["step"] == 1
    assert np.array_equal(st["m"], keep[2]["m"]) and np.array_equal(st["v"], keep[2]["v"])
    loss, td = a.train(*args)
    assert np.isfinite(loss) and td.shape == (4,) and a._engine.get_opt_state()["step"] == 2
    a.set_n_step(5)                     # no change: the engine stays
    assert a._engine is not None
