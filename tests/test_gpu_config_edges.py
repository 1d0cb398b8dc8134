"""-m gpu: the learners against their float64 oracles at the configurations the project runs, benchmarks or accepts
but the other parity tests do not reach, with the same bars (1e-4 relative, 1e-3 on the applied update, the kink and
argmax rules of tests/parity.py and tests/apex_parity.py):

* IMPALA at the per-GPU batch sizes of ``bench.py --scaling strong`` (B = 64 / 128 / 256, M = B * T rows up to 5120):
  every split-K plan and GEMM grid that depends on M;
* num_action = 32, the largest accepted value in all four families (full 32-wide dlogits / dq rows, kMaxA);
* the stand-alone ``from_softmax`` on both sides of its shared-memory fast-path boundary;
* the optimizer tails: global-norm clipping engaged, the polynomial learning-rate decay reaching its end value, and an
  optimizer state restored mid-training;
* the R2D2 benchmark shape (seq_len 80, burn_in 40: a loss window Nt = 39 > 32, two window steps per lane);
* the ``grad_scale`` of a data-parallel update, emulated with two handles on one GPU;
* the act / td-error entry points at their largest n.

Every case asserts that it reached its edge (grad_norm > clip, the lr sequence, Nt > 32, the row or n count)."""
import numpy as np
import pytest
import torch

import a3c_parity as a3p
import apex_parity as ap
import parity
import r2d2_parity as rp
from oracle import a3c_torch as at
from oracle import apex_torch as ax
from oracle import impala_torch as it
from oracle import r2d2_torch as rt
from oracle import vtrace_np

pytestmark = pytest.mark.gpu


def _impala(errs):          # also the A3C bar
    bad = parity.failures(errs)
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:12]


def _apex(errs):
    bad = ap.apex_failures(errs)
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:12]


def _r2d2(errs):
    bad = rp.r2d2_failures(errs)
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:12]


# the learning-rate schedule of the decay cases: learning_frame = 2 reaches the end value at step 2
DECAY = dict(start_learning_rate=6e-4, end_learning_rate=1e-4, learning_frame=2)


def _assert_decay_sequence(trace):
    """The lr of steps 0..3 (pre-increment global step) is start, midpoint, end, end in float32."""
    lr = [float(o["learning_rate"]) for o in trace]
    s, e = float(np.float32(DECAY["start_learning_rate"])), float(np.float32(DECAY["end_learning_rate"]))
    assert len(lr) == 4
    assert abs(lr[0] - s) < 1e-9 and abs(lr[1] - 0.5 * (s + e)) < 1e-9 and lr[2] == lr[3] and abs(lr[3] - e) < 1e-9, lr


# ---- IMPALA at the benchmarked batch sizes ---------------------------------------------------------------------------
@pytest.mark.parametrize("B", [64, 128])
def test_impala_benchmark_batch_layers(native, B):
    """Per-GPU batch of bench.py --scaling strong on 4 / 2 GPUs, with activations and da1..da3 compared too."""
    assert B * 20 > 640                       # beyond the largest M of tests/test_gpu_learner.py
    _impala(parity.compare_step(B, T=20, A=18, layers=True))


def test_impala_benchmark_batch_256(native):
    """One GPU of bench.py --scaling strong: M = 5120 rows."""
    assert 256 * 20 == 5120
    _impala(parity.compare_step(256, T=20, A=18, layers=False))


def test_impala_benchmark_batch_64_mode2(native):
    """The same shape through the 3xTF32 wgmma path (math mode 2), as a cross-check of the default mode 5."""
    _impala(parity.compare_step(64, T=20, A=18, layers=False, math_mode=2))


def test_impala_longest_trajectory_batch_32(native):
    """T = 32 (the largest accepted) at B = 32: M = 1024, Mb = 960 rows of gradient."""
    assert 32 * 32 == 1024
    _impala(parity.compare_step(32, T=32, A=18, layers=False))


def test_impala_conv_data_gradients_batch_128(native):
    """The conv3 / conv2 data gradients in isolation (tests/test_gpu_conv_dgrad.py) at B = 128: Mb = 2304 rows."""
    from test_gpu_conv_dgrad import check_conv_data_gradients
    check_conv_data_gradients(128, 20, 18)


# ---- IMPALA at num_action = 32 ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [5, 1])
def test_impala_max_actions_max_trajectory(native, mode):
    """T = 32 and A = 32 together: both at their accepted maximum."""
    _impala(parity.compare_step(3, T=32, A=32, math_mode=mode))


def test_impala_max_actions_cuda_graph(native):
    _impala(parity.compare_step(4, T=20, A=32, steps=2, layers=False, use_cuda_graph=True))


def test_impala_max_actions_fused_vtrace(native):
    """The fused V-trace / loss kernel's taps (tests/test_gpu_vtrace_property.py) with the lane-per-action softmax full."""
    from test_gpu_vtrace_property import check_fused_learner_vtrace
    check_fused_learner_vtrace(5, 20, 32, 1234, "soft_asymmetric")


# ---- stand-alone from_softmax at its fast-path boundary ----------------------------------------------------------------
def _softmax(x):
    e = np.exp(x - x.max(-1, keepdims=True))
    return (e / e.sum(-1, keepdims=True)).astype(np.float32)


@pytest.mark.parametrize("B,T,A,pipe", [(40, 32, 24, True), (40, 32, 25, False), (40, 32, 32, False),
                                         (37, 7, 5, False)])
def test_from_softmax_fast_path_boundary(native, B, T, A, pipe):
    """vtrace.cu launch_fs: the cp.async pipe kernel takes T <= 32, T * A % 4 == 0 and 4 warps x 4 x T x A floats of
    shared memory <= 48 KB; T = 32, A = 24 is exactly 48 KB.  A = 25 / 32 and T * A = 35 take the chunked kernel."""
    smem = 4 * 4 * T * A * 4
    assert (T <= 32 and (T * A) % 4 == 0 and smem <= 48 * 1024) == pipe
    from distributed_reinforcement_learning_b200.optimizer import vtrace
    rng = np.random.default_rng(B * 1000 + A)
    mu, pi = _softmax(rng.standard_normal((B, T, A))), _softmax(rng.standard_normal((B, T, A)) * 2.0)
    act = rng.integers(0, A, (B, T)).astype(np.int32)
    disc = ((rng.random((B, T)) >= 0.1) * 0.99).astype(np.float32)
    rew, val, nval = (rng.standard_normal((B, T)).astype(np.float32) for _ in range(3))
    vs, rho = vtrace.from_softmax(mu, pi, act, disc, rew, val, nval, A)
    f = lambda x: x.astype(np.float64)     # noqa: E731
    evs, erho = vtrace_np.from_softmax(f(mu), f(pi), act, f(disc), f(rew), f(val), f(nval), A)
    assert parity.rel_err(vs, evs) < parity.TOL and parity.rel_err(rho, erho) < parity.TOL


# ---- IMPALA optimizer (RMSProp) --------------------------------------------------------------------------------------
@pytest.mark.parametrize("clip", [1e6, 1.0])
def test_impala_gradient_clip(native, clip):
    """1e6: never engaged (the update is the raw gradient's); 1.0: engaged on every step."""
    trace = []
    _impala(parity.compare_step(4, T=20, steps=2, layers=False, opt=dict(gradient_clip_norm=clip), trace=trace))
    gn = [o["grad_norm"] for o in trace]
    assert all(g > clip for g in gn) if clip == 1.0 else all(g < clip for g in gn), gn


def test_impala_learning_rate_decay(native):
    trace = []
    _impala(parity.compare_step(2, T=5, steps=4, layers=False, opt=DECAY, trace=trace))
    _assert_decay_sequence(trace)


def test_impala_restored_optimizer_state(native):
    """Random positive RMSProp slots and global step 1e7 of learning_frame 2e7: the float32 step / decay arithmetic
    gives lr = start / 2 and the step counter continues from 1e7."""
    A = 18
    ms = np.random.default_rng(3).uniform(0.05, 2.0, it.param_count(num_action=A)).astype(np.float32)
    trace = []
    _impala(parity.compare_step(2, T=5, A=A, steps=2, layers=False, opt=dict(learning_frame=2e7),
                                init_state=dict(ms=ms, step=10 ** 7), trace=trace))
    assert [o["step"] for o in trace] == [10 ** 7 + 1, 10 ** 7 + 2]
    assert abs(trace[0]["learning_rate"] - float(np.float32(6e-4)) / 2) < 1e-9      # the default start rate / 2


# ---- Ape-X and A3C -----------------------------------------------------------------------------------------------------
def _adam_state(n, seed):
    """A mid-training Adam state: m ~ N(0, 1e-4), v in [1e-10, 1e-6], beta powers after 1000 updates, step 1e6."""
    rng = np.random.default_rng(seed)
    return dict(m=(rng.standard_normal(n) * 1e-4).astype(np.float32),
                v=rng.uniform(1e-10, 1e-6, n).astype(np.float32), step=10 ** 6,
                beta1_power=float(np.float32(0.9 ** 1000)), beta2_power=float(np.float32(0.999 ** 1000)))


FAMILIES = {"apex": (ap.compare_step, _apex, ax.param_count), "a3c": (a3p.compare_step, _impala, at.param_count)}


@pytest.mark.parametrize("family", ["apex", "a3c"])
@pytest.mark.parametrize("B,A", [(64, 4), (100, 4), (5, 32)])
def test_adam_learner_shapes(native, family, B, A):
    """B = 64 / 100 (128 / 200 rows through the network, main and next state) and A = 32."""
    compare, check, _ = FAMILIES[family]
    check(compare(B, A=A))


@pytest.mark.parametrize("family", ["apex", "a3c"])
def test_adam_learner_gradient_clip(native, family):
    compare, check, _ = FAMILIES[family]
    trace = []
    check(compare(4, A=4, steps=2, opt=dict(gradient_clip_norm=0.5), trace=trace))
    assert all(o["grad_norm"] > 0.5 for o in trace), [o["grad_norm"] for o in trace]


@pytest.mark.parametrize("family", ["apex", "a3c"])
def test_adam_learner_learning_rate_decay(native, family):
    compare, check, _ = FAMILIES[family]
    trace = []
    check(compare(3, A=4, steps=4, opt=DECAY, trace=trace))
    _assert_decay_sequence(trace)


@pytest.mark.parametrize("family", ["apex", "a3c"])
def test_adam_learner_restored_state(native, family):
    compare, check, count = FAMILIES[family]
    st = _adam_state(count(num_action=4), 11)
    trace = []
    check(compare(4, A=4, steps=2, init_state=st, trace=trace))
    assert [o["step"] for o in trace] == [10 ** 6 + 1, 10 ** 6 + 2]


# ---- R2D2 ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [2, 1])
def test_r2d2_benchmark_shape(native, mode):
    """tools/bench_r2d2.py: B = 16, seq_len 80, burn_in 40 -> Nt = 39 loss steps, two per lane of r2d2_td_kernel."""
    assert 80 - 40 - 1 > 32
    _r2d2(rp.compare_step(16, S=80, bi=40, A=4, C=1, math_mode=mode))


def test_r2d2_window_of_three_iterations(native):
    """burn_in 0 at seq_len 80: Nt = 79, three window steps per lane."""
    assert 80 - 0 - 1 > 64
    _r2d2(rp.compare_step(4, S=80, bi=0, A=6, C=4))


def test_r2d2_done_heavy(native):
    """Half of the steps terminal, and every sequence terminal at t = 0 and t = S - 1: the LSTM state resets inside the
    burn-in, inside the window and on its last step."""
    b = rp.make_batch(3, 20, 4, 1, 2468, done_rate=0.5, done_ends=True)
    assert b["done"][:, 0].all() and b["done"][:, -1].all() and 0.4 < b["done"].mean() < 0.8
    _r2d2(rp.compare_step(3, S=20, bi=5, done_rate=0.5, done_ends=True))


def test_r2d2_max_actions(native):
    _r2d2(rp.compare_step(3, S=9, bi=2, A=32))


def test_r2d2_restored_state_and_learning_rate(native):
    n = rt.param_count(num_action=4, lstm_size=64, input_shape=(84, 84, 1))
    trace = []
    _r2d2(rp.compare_step(3, S=8, bi=3, steps=2, opt=dict(learning_rate=3e-4), init_state=_adam_state(n, 12),
                          trace=trace))
    assert [o["step"] for o in trace] == [10 ** 6 + 1, 10 ** 6 + 2]


# ---- data parallelism emulated on one GPU ------------------------------------------------------------------------------
def _dp_case(family, clip):
    """-> (make(Bn) -> engine, whole minibatch, stage(engine, batch))."""
    if family == "r2d2":
        from distributed_reinforcement_learning_b200.r2d2_learner import NativeR2D2Learner
        kwp = dict(num_action=4, lstm_size=64, input_shape=(84, 84, 1))
        pm = rt.flatten_params(rt.init_params(0, torch.float32, **kwp))
        pt = rt.flatten_params(rt.init_params(1, torch.float32, **kwp))

        def make(Bn):
            e = NativeR2D2Learner(batch=Bn, seq_len=10, burn_in=3)
            e.set_params(pm, 0)
            e.set_params(pt, 1)
            return e

        def stage(e, b):
            e.stage(0, b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"], b["done"],
                    b["weight"])
        return make, rt.make_sequences(6, S=10, seed=41), stage
    opt = {} if clip is None else dict(gradient_clip_norm=clip)
    pm = ax.flatten_params(ax.init_params(0, torch.float32, num_action=4))
    batch = ax.make_transitions(8, seed=41)
    if family == "apex":
        from distributed_reinforcement_learning_b200.apex_learner import NativeApexLearner
        pt = ax.flatten_params(ax.init_params(1, torch.float32, num_action=4))

        def make(Bn):
            e = NativeApexLearner(batch=Bn, num_action=4, **opt)
            e.set_params(pm, 0)
            e.set_params(pt, 1)
            return e

        def stage(e, b):
            e.stage(0, *[b[k] for k in ax.TRAIN_FIELDS])
        return make, batch, stage
    from distributed_reinforcement_learning_b200.a3c_learner import NativeA3CLearner

    def make(Bn):
        e = NativeA3CLearner(batch=Bn, num_action=4, **opt)
        e.set_params(pm)
        return e

    def stage(e, b):
        e.stage(0, *[b[k] for k in at.TRAIN_FIELDS])
    return make, batch, stage


def _scalars(out):
    out = out[0] if isinstance(out, tuple) else out
    return np.array([out[k] for k in sorted(out) if k not in ("step", "learning_rate")], np.float64)


@pytest.mark.parametrize("family,clip", [("apex", None), ("a3c", None), ("r2d2", None), ("apex", 0.5), ("a3c", 0.5)])
def test_data_parallel_grad_scale_on_one_gpu(native, family, clip):
    """Two handles on device 0 with half of the minibatch each: forward_backward on both, handle 1's gradient bucket
    (loss sums in its tail) added into handle 0's on its stream, then apply(grad_scale = 1/2) -- the data-parallel update
    of dp.py without a second GPU.  It must equal one handle stepping on the whole minibatch: the bucket is the sum of
    two half-batch MEAN gradients, and grad_scale enters both the global norm and the clip scale."""
    import ctypes as C

    from distributed_reinforcement_learning_b200 import _native as N
    make, batch, stage = _dp_case(family, clip)
    n = len(batch["reward"]) // 2
    halves = [{k: v[i * n:(i + 1) * n] for k, v in batch.items()} for i in range(2)]
    h0, h1 = make(n), make(n)
    try:
        p0 = h0.get_params()
        stage(h0, halves[0])
        stage(h1, halves[1])
        N.check(h0._fn("forward_backward")(h0._h, 0))
        N.check(h1._fn("forward_backward")(h1._h, 0))
        b0, b1 = h0._dp._tensor(), h1._dp._tensor()
        h1._dp._stream.synchronize()
        with torch.cuda.stream(h0._dp._stream):       # ordered after h0's backward, before its apply
            b0.add_(b1)
        N.check(h0._fn("apply")(h0._h, C.c_float(0.5)))
        out = h0.wait()
        st, g, p = h0.get_opt_state(), h0.get_grads(), h0.get_params()
    finally:
        h0.close()
        h1.close()
    full = make(2 * n)
    try:
        stage(full, batch)
        out1 = full.step(0)
        st1, g1, p1 = full.get_opt_state(), full.get_grads(), full.get_params()
    finally:
        full.close()
    o1 = out1[0] if isinstance(out1, tuple) else out1
    if clip is not None:
        assert o1["grad_norm"] > clip
    # the tolerances of test_gpu_multi.py::test_two_gpu_mean_loss_learners_equal_single_replica
    assert parity.rel_err(0.5 * g, g1) < parity.TOL
    assert parity.rel_err(st["m"], st1["m"]) < parity.TOL and parity.rel_err(st["v"], st1["v"]) < 2 * parity.TOL
    assert np.allclose(_scalars(out), _scalars(out1), rtol=1e-4)
    d = np.abs((p - p0) - (p1 - p0))
    assert np.quantile(d, 0.999) <= 1e-2 * np.max(np.abs(p1 - p0)) and np.max(d) <= 2.1 * np.max(np.abs(p1 - p0))


# ---- act / td-error at their n limits ------------------------------------------------------------------------------------
def test_impala_act_at_n_limit(native):
    """drl_learner_act accepts n <= B * T single-step forwards; n = B * T = 80, and n + 1 is refused."""
    from distributed_reinforcement_learning_b200 import _native as N
    B, T, A = 4, 20, 18
    batch, params, cfg = parity.make_case(B, T, A, seed=6)
    n = B * T
    st = batch["state"].reshape((n, 84, 84, 4))
    pa = batch["previous_action"].reshape(n)
    h0, c0 = batch["initial_h"].reshape(n, 256), batch["initial_c"].reshape(n, 256)
    eng = parity.native_learner(batch, params, cfg)
    try:
        pol, h, c = eng.act(st, pa, h0, c0)
        with pytest.raises(N.DrlError):
            eng.act(np.concatenate([st, st[:1]]), np.concatenate([pa, pa[:1]]), np.concatenate([h0, h0[:1]]),
                    np.concatenate([c0, c0[:1]]))
    finally:
        eng.close()
    p64 = {k: v.double() for k, v in params.items()}
    x = torch.from_numpy((st.astype(np.float64) / 255).astype(np.float32)).double()
    a, v, cc, hh = it.network(p64, x, torch.from_numpy(pa.astype(np.int64)), torch.from_numpy(h0).double(),
                              torch.from_numpy(c0).double(), A, 256)
    assert pol.shape == (n, A)
    assert parity.rel_err(pol, a.numpy()) < parity.TOL
    assert parity.rel_err(h, hh.numpy()) < parity.TOL and parity.rel_err(c, cc.numpy()) < parity.TOL


def test_apex_act_at_n_limit(native):
    """drl_apex_act accepts n <= 2B (the main and the next states of a minibatch); n = 2B = 12."""
    A, B = 4, 6
    params, target = ax.init_params(0, torch.float32, num_action=A), ax.init_params(1, torch.float32, num_action=A)
    L = ax.Learner(params, target, torch.float64, num_action=A)
    b = ax.make_transitions(B, A=A, seed=8)
    st = np.concatenate([b["state"], b["next_state"]])
    pa = np.concatenate([b["previous_action"], b["action"]])
    eng = ap.native_apex(B, A, params, target)
    try:
        q = eng.act(st, pa)
    finally:
        eng.close()
    assert q.shape == (2 * B, A)
    assert parity.rel_err(q, L.main_q(st, pa).numpy()) < parity.TOL


def test_r2d2_act_and_td_error_at_n_limit(native):
    """drl_r2d2_act accepts n <= B * S single steps (n = 24 here) and drl_r2d2_td_error n <= B sequences (n = B = 3)."""
    A, S, bi, B = 4, 8, 3, 3
    kwp = dict(num_action=A, lstm_size=64, input_shape=(84, 84, 1))
    params, target = rt.init_params(0, torch.float32, **kwp), rt.init_params(1, torch.float32, **kwp)
    L = rt.Learner(params, target, torch.float64, seq_len=S, burn_in=bi, **kwp)
    b = rt.make_sequences(B, S=S, A=A, seed=9)
    n = B * S
    st, pa = b["state"].reshape((n, 84, 84, 1)), b["previous_action"].reshape(n)
    hh, cc = b["h"].reshape(n, 64), b["c"].reshape(n, 64)
    eng = rp.native_r2d2(B, S, bi, A, 1, params, target)
    try:
        q, h2, c2 = eng.act(st, pa, hh, cc)
        td = eng.td_error(b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"],
                          b["done"])
    finally:
        eng.close()
    rq, rh, rc = L.step_q(st, hh, cc, pa)
    assert q.shape == (n, A)
    assert parity.rel_err(q, rq) < parity.TOL and parity.rel_err(h2, rh) < parity.TOL and parity.rel_err(c2, rc) < parity.TOL
    ref = [L.get_td_error(*[b[k][i] for k in rt.TRAIN_FIELDS[:-1]]) for i in range(B)]
    assert td.shape == (B,) and parity.rel_err(td, np.asarray(ref)) < parity.TOL
