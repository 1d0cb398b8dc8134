"""The IMPALA learner's recurrent mode on the GPU (``NativeLearner(..., recurrent=True)``, DESIGN.md section 21): full
steps against the float64 recurrent oracle (tests/impala_recurrent_oracle.py) at the 1e-4 bar, the recurrence and BPTT
kernels each against a float64 reference fed from the step's own buffers, and the identities -- on-policy trajectories
give the stored-state learner's losses, repeated / graph / eager / split steps are bit-equal, and train_from_queue is
train."""
import numpy as np
import pytest
import torch

from oracle import impala_torch as it
from oracle import synthetic

import impala_recurrent_oracle as ro
import parity

pytestmark = pytest.mark.gpu

EPS32 = 2.0 ** -24
K_X = 3136 + 256


@pytest.fixture(scope="module")
def gpu(native):
    if native.device_count() < 1:
        pytest.skip("needs a CUDA device")
    return native


def _check(errs):
    bad = ro.failures(errs)
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:10]


@pytest.mark.parametrize("B,T,A,mode,graph", [
    (4, 20, 18, 5, True), (32, 20, 18, 5, True), (4, 3, 18, 5, True), (4, 32, 18, 5, True), (4, 20, 32, 5, True),
    (4, 20, 18, 5, False), (4, 20, 18, 2, True), (4, 20, 18, 2, False), (9, 7, 18, 2, True)])
def test_step_matches_float64_recurrent_oracle(gpu, B, T, A, mode, graph):
    _check(ro.compare_step(B, T, A, math_mode=mode, use_cuda_graph=graph))


@pytest.mark.parametrize("mode", [5, 2])
def test_three_steps_match_float64_recurrent_oracle(gpu, mode):
    """three consecutive steps: the RMSProp slots and the parameters the second and third steps run on"""
    _check(ro.compare_step(4, 20, 18, steps=3, math_mode=mode))


def test_no_dones_and_dones_everywhere(gpu):
    _check(ro.compare_step(4, 8, 18, dones=[]))
    _check(ro.compare_step(3, 8, 18, dones=[(b, t) for b in range(3) for t in range(8)]))


# ---- per kernel ---------------------------------------------------------------------------------------------------
def _case(B=32, T=20, A=18, seed=21, graph=True):
    batch, params, cfg = parity.make_case(B, T, A, seed)
    batch = ro.with_dones(batch, ro.default_dones(B, T))
    eng = parity.native_learner(batch, params, cfg, recurrent=True, use_cuda_graph=graph)
    eng.stage(0, *[batch[k] for k in synthetic.TRAIN_FIELDS])
    p = {k: v.double().numpy() for k, v in params.items()}
    return eng, batch, p


def _rows(eng, name, M, n):
    return eng.read_buffer(name, M * n).astype(np.float64).reshape(M, n)


def _where(m, col, B):
    """the (t, b) of row m, and the cluster / CTA rank that computed column `col` of it (8 trajectories per cluster,
    32 hidden units per CTA)"""
    t, b = divmod(m, B)
    return "t=%d b=%d cluster %d CTA rank %d" % (t, b, b // 8, (col % 256) // 32)


def test_recurrence_kernel_against_float64_reference(gpu):
    """lstm_unroll_fwd: gates from [a3 | emb] W_x + b + h_in W_h, the cell update, and the state each step reads (the
    previous output, or the recorded state after a done), fed from the step's own buffers.  Per-element bound: the
    pre-activation is a sum of 3648 products, |error| <= 2 * 3648 * 2^-24 * sum |terms|; the activations do not
    enlarge it; the cell update adds a few roundings."""
    B, T, A = 32, 20, 18
    eng, batch, p = _case(B, T, A)
    try:
        eng.forward(0)
        M = B * T
        a3 = _rows(eng, "a3", M, 3136)
        table = eng.read_buffer("emb", A * 256).astype(np.float64).reshape(A, 256)
        pa = parity.to_time_major(batch["previous_action"])
        hin, cin = _rows(eng, "hin", M, 256), _rows(eng, "cin", M, 256)
        hout, c1, tc = _rows(eng, "hout", M, 256), _rows(eng, "c1", M, 256), _rows(eng, "tc", M, 256)
        gates = _rows(eng, "gates", M, 1024)
    finally:
        eng.close()
    x = np.concatenate([a3, table[pa]], axis=1)
    W, b = p["lstm.w"], p["lstm.b"]
    pre = x @ W[:K_X] + hin @ W[K_X:] + b
    scale = np.abs(x) @ np.abs(W[:K_X]) + np.abs(hin) @ np.abs(W[K_X:]) + np.abs(b)
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))
    ref = np.concatenate([sig(pre[:, :256]), np.tanh(pre[:, 256:512]), sig(pre[:, 512:768] + 1.0),
                          sig(pre[:, 768:])], axis=1)
    bound = 2 * 3648 * EPS32 * scale + 4 * EPS32
    bad = np.argwhere(np.abs(gates - ref) > bound)
    assert bad.size == 0, ["gates %s: %.3g > %.3g" % (_where(m, c, B), abs(gates[m, c] - ref[m, c]), bound[m, c])
                           for m, c in bad[:8]]
    si, tj, sf, so = gates[:, :256], gates[:, 256:512], gates[:, 512:768], gates[:, 768:]
    c_ref = sf * cin + si * tj
    bad = np.argwhere(np.abs(c1 - c_ref) > 4 * EPS32 * (np.abs(sf * cin) + np.abs(si * tj)) + 1e-30)
    assert bad.size == 0, ["c %s" % _where(m, u, B) for m, u in bad[:8]]
    bad = np.argwhere(np.abs(tc - np.tanh(c1)) > 4 * EPS32 + 1e-30)
    assert bad.size == 0, ["tanh c %s" % _where(m, u, B) for m, u in bad[:8]]
    bad = np.argwhere(np.abs(hout - so * tc) > 2 * EPS32 * np.abs(so * tc) + 1e-30)
    assert bad.size == 0, ["h %s" % _where(m, u, B) for m, u in bad[:8]]
    # the state each step read: exactly the recorded one at t = 0 and after a done, else exactly the previous output
    h_rec, c_rec = parity.to_time_major(batch["initial_h"]), parity.to_time_major(batch["initial_c"])
    done = batch["done"]
    for m in range(M):
        t, bb = divmod(m, B)
        restart = t == 0 or done[bb, t - 1]
        want_h = h_rec[m] if restart else hout[m - B]
        want_c = c_rec[m] if restart else c1[m - B]
        assert np.array_equal(hin[m], want_h) and np.array_equal(cin[m], want_c), \
            "state entering %s (restart %s)" % (_where(m, 0, B), restart)


def test_bptt_kernel_against_float64_reference(gpu):
    """lstm_unroll_bwd: dz of the T - 2 steps with loss gradient, from the heads' dL/dh (two partials), the forward's
    gates / tanh c / c_in, and dL/dh_in of the next step formed from the kernel's own dz of that step (no carry across a
    done).  Per-element bound: dh_in is a sum of 1024 products, |error| <= 2 * 1024 * 2^-24 * sum |terms|, plus 1e-5 of
    the row's largest |dz| for the c gradient the kernel carries in float32 through at most 29 steps."""
    B, T, A = 32, 20, 18
    eng, batch, p = _case(B, T, A, seed=22)
    try:
        eng.forward_backward(0)
        M, Mb = B * T, B * (T - 2)
        dhp = eng.read_buffer("dh_part", 2 * Mb * 256).astype(np.float64).reshape(2, Mb, 256)
        gates = _rows(eng, "gates", M, 1024)
        tc, cin = _rows(eng, "tc", M, 256), _rows(eng, "cin", M, 256)
        dz = _rows(eng, "dz", Mb, 1024)
    finally:
        eng.close()
    Wh = p["lstm.w"][K_X:]
    done = batch["done"]
    dc_carry = np.zeros((B, 256))
    for t in range(T - 3, -1, -1):
        rows = slice(t * B, (t + 1) * B)
        keep = (~done[:, t]).astype(np.float64)[:, None]
        dh = dhp[0, rows] + dhp[1, rows]
        scale = np.zeros_like(dh)
        if t + 1 < T - 2:
            nxt = dz[(t + 1) * B:(t + 2) * B]
            dh = dh + keep * (nxt @ Wh.T)
            scale = keep * (np.abs(nxt) @ np.abs(Wh).T)
        g = gates[rows]
        si, tj, sf, so = g[:, :256], g[:, 256:512], g[:, 512:768], g[:, 768:]
        tcv, cprev = tc[rows], cin[rows]
        d_o = dh * tcv * so * (1 - so)
        dc = keep * dc_carry + dh * so * (1 - tcv * tcv)
        ref = np.concatenate([dc * tj * si * (1 - si), dc * si * (1 - tj * tj), dc * cprev * sf * (1 - sf), d_o], axis=1)
        dc_carry = dc * sf
        got = dz[rows]
        bound = 2 * 1024 * EPS32 * np.tile(scale, 4) + 1e-5 * np.max(np.abs(ref), axis=1, keepdims=True) + 1e-30
        bad = np.argwhere(np.abs(got - ref) > bound)
        assert bad.size == 0, ["dz %s: %.3g > %.3g" % (_where(t * B + r, c, B), abs(got[r, c] - ref[r, c]), bound[r, c])
                               for r, c in bad[:8]]


# ---- identities ---------------------------------------------------------------------------------------------------
def _train_args(batch):
    return [batch[k] for k in synthetic.TRAIN_FIELDS]


def _run(batch, params, cfg, steps=2, split=False, **kw):
    eng = parity.native_learner(batch, params, cfg, recurrent=True, **kw)
    outs = []
    try:
        for s in range(steps):
            eng.stage(s % 2, *_train_args(batch))
            if split:
                eng.forward_backward(s % 2)
                eng.apply()
                outs.append(eng.wait())
            else:
                outs.append(eng.step(s % 2))
        return outs, eng.get_grads(), eng.get_params(), eng.get_opt_state()[0]
    finally:
        eng.close()


@pytest.mark.parametrize("mode", [5, 2])
def test_repeated_graph_eager_and_split_steps_are_bit_equal(gpu, mode):
    batch, params, cfg = parity.make_case(8, 20, 18, seed=31)
    batch = ro.with_dones(batch, ro.default_dones(8, 20))
    ref = _run(batch, params, cfg, math_mode=mode, use_cuda_graph=True)
    for kw in (dict(use_cuda_graph=True), dict(use_cuda_graph=False), dict(use_cuda_graph=True, split=True),
               dict(use_cuda_graph=False, split=True)):
        got = _run(batch, params, cfg, math_mode=mode, **kw)
        assert got[0] == ref[0], kw
        for a, b in zip(got[1:], ref[1:]):
            assert np.array_equal(a, b), kw


def test_on_policy_trajectories_give_the_stored_state_losses(gpu):
    """Trajectories recorded by NativePolicy through a VectorActor with life-loss environments under parameters P,
    trained by learners holding P: the recurrent learner recomputes the states the actor recorded, so its losses are
    the stored-state learner's within 1e-4 relative."""
    import test_gpu_impala_queue as q
    P = q._params()
    hq, _, _, _ = q._arms(32, unrolls=1, params=P)
    b = hq.sample_batch()
    args = [np.asarray(v) for v in (b.state, b.reward, b.action, b.done, b.behavior_policy, b.previous_action,
                                    b.previous_h, b.previous_c)]
    assert np.asarray(b.done).any()
    from distributed_reinforcement_learning_b200.learner import NativeLearner
    out = {}
    for rec in (False, True):
        eng = NativeLearner(batch=32, trajectory=q.T, num_action=q.A, recurrent=rec)
        try:
            eng.set_params(P)
            eng.stage(0, *args)
            out[rec] = eng.step(0)
        finally:
            eng.close()
    for k in ("pi_loss", "baseline_loss", "entropy", "total_loss"):
        assert parity.rel_err(out[True][k], out[False][k]) <= 1e-4, (k, out[True][k], out[False][k])


@pytest.mark.parametrize("graph", [True, False])
def test_train_from_queue_is_bitwise_train(gpu, graph):
    import test_gpu_impala_queue as q
    params = q._params()
    hq, dq, _, _ = q._arms(32, unrolls=2, params=params)
    ag_h, ag_d = q._agent(params, "rq_host_%d" % graph, graph), q._agent(params, "rq_dev_%d" % graph, graph)
    ag_h.set_recurrent(True)
    ag_d.set_recurrent(True)
    for _ in range(2):
        b = hq.sample_batch()
        rh = ag_h.train(b.state, b.reward, b.action, b.done, b.behavior_policy, b.previous_action, b.previous_h,
                        b.previous_c)
        rd = ag_d.train_from_queue(dq)
        assert rh == rd
        assert np.isfinite(rd).all()
    assert ag_h._engine.recurrent and ag_d._engine.recurrent
    assert np.array_equal(ag_h._engine.get_params(), ag_d._engine.get_params())


def test_checkpoints_load_across_modes_and_act_stays_one_step(gpu, tmp_path):
    """save_weights in one mode, load_weights in the other: the same parameters; drl_learner_act is the single step
    of the stored-state mode in both."""
    import test_gpu_impala_queue as q
    params = q._params()
    a = q._agent(params, "ck_rec", True)
    a.set_recurrent(True)
    b = q._agent(params, "ck_plain", True)
    batch, _, _ = parity.make_case(4, 20, 18, seed=41)
    a.train(*_train_args(batch))
    a.save_weights(str(tmp_path / "w"))
    b.load_weights(str(tmp_path / "w"))
    b.train(*_train_args(batch))
    assert b._engine.get_params().size == a._engine.get_params().size
    a._pull_state()
    np.testing.assert_array_equal(np.load(str(tmp_path / "w.npz"))["params"], a._params)
    st = batch["state"][:, 0]
    pa, h, c = batch["previous_action"][:, 0], batch["initial_h"][:, 0], batch["initial_c"][:, 0]
    p = a._engine.get_params()
    b._engine.set_params(p)
    ra, rb = a._engine.act(st, pa, h, c), b._engine.act(st, pa, h, c)
    for x, y in zip(ra, rb):
        assert np.array_equal(x, y)
