"""-m gpu: every kernel of the Ape-X, A3C and R2D2 learner steps checked on its own, against a float64 reference
computed from the buffers that kernel read in the same step (tests/adam_layer_parity.py; its references are checked
against the float64 oracle by tests/test_oracle_adam_layer_local.py).  Same metric, per-block reporting and failure
message as tests/test_gpu_layer_local.py; the R2D2 recurrence is held per element to layer_parity.lstm_bounds with the
K = 64 FFMA dot product as the pre-activation bar (at lstm_size 256 / 512: a per-element bound from the cluster
kernel's summation order, and the BPTT's o block per element), the loss kernels per element to the rounding bounds of
the values they combine, and the recurrence's state hand-over and the gradient rows outside the loss window bitwise.

Case matrix, math mode 2 (3xTF32, the default) unless noted:
  * R2D2 (B, S, burn_in, A, C) from init at the reference config, the benchmark shape (Nt = 39 > 32: the TD kernel's
    lane loop; B > 8: its warp loop), M = 2 (partial tiles everywhere), A = 32 and B = 140 (more recurrence CTAs than
    SMs); trained, done-heavy, large-return and exact next-q tie steps at the reference config; saturated gates at
    the benchmark shape;
    math mode 1 at the reference config and the benchmark shape.
  * R2D2 at lstm_size 256 and 512 (the cluster recurrence, csrc/r2d2_cluster.cuh) from init at the reference config,
    the benchmark shape, M = 2 (one chunk with R - 1 dead sequences), A = 32 with a partial last chunk, and "many
    chunks": S = 3 and a B computed from recurrence_clusters() so that every cluster of the forward and the BPTT walks
    more than one chunk of R sequences and the last chunk is partial; trained at the reference config and saturated
    gates at the benchmark shape at both widths, done-heavy, large-return and tie steps at 512; math mode 1 at the
    reference config and the benchmark shape; the forward of td_error calls over 1 and R + 1 sequences.
  * Ape-X and A3C at B = 1, 32 and 300 (n > 256: the loss kernels' block-stride loop) with A = 4 and 18 from init;
    trained, large returns (Ape-X, reward_clipping "none"), exact next-q ties (Ape-X) and a peaked policy (A3C);
    math mode 1 at two shapes.
Every case asserts that it reached its regime."""
import functools

import numpy as np
import pytest

import adam_layer_parity as alp

pytestmark = pytest.mark.gpu

R2D2_SHAPES = [(16, 15, 7, 4, 1),     # the reference config
               (16, 80, 40, 4, 1),    # the benchmark shape
               (1, 2, 0, 2, 4),       # M = 2
               (5, 7, 5, 32, 4),      # A = 32
               (140, 4, 1, 4, 1)]     # more sequences than SMs
# lstm_size 256 / 512: B = MANY is computed at run time (many_chunks_B) so that clusters walk several chunks
MANY = "many"
WIDE_SHAPES = R2D2_SHAPES[:4] + [(MANY, 3, 1, 4, 1)]
WIDTHS = (256, 512)
R2D2_CASES = [(2,) + s + (64, "init") for s in R2D2_SHAPES] + \
             [(2,) + R2D2_SHAPES[0] + (64, r) for r in ("trained", "done_heavy", "large_returns", "ties")] + \
             [(2,) + R2D2_SHAPES[1] + (64, "saturated")] + \
             [(1,) + s + (64, "init") for s in R2D2_SHAPES[:2]]
R2D2_CASES += [(2,) + s + (L, "init") for L in WIDTHS for s in WIDE_SHAPES] + \
              [(2,) + R2D2_SHAPES[0] + (512, r) for r in ("trained", "done_heavy", "large_returns", "ties")] + \
              [(2,) + R2D2_SHAPES[0] + (256, "trained")] + \
              [(2,) + R2D2_SHAPES[1] + (L, "saturated") for L in WIDTHS] + \
              [(1,) + s + (L, "init") for L in WIDTHS for s in R2D2_SHAPES[:2]]


def _r2d2_id(case):
    """The parameter id; the lstm_size 64 cases keep the ids they had before the width was a parameter."""
    mode, B, S, bi, A, C, L, regime = case
    return "-".join(str(x) for x in (mode, B, S, bi, A, C) + (() if L == 64 else ("L%d" % L,)) + (regime,))


@functools.lru_cache(maxsize=None)
def recurrence_plan(L):
    """(R, P_fwd, P_bwd) at width L: sequences per cluster pass (the library's plan) and the clusters of the forward /
    BPTT recurrence the device places at once (recurrence_clusters())."""
    from distributed_reinforcement_learning_b200.r2d2_learner import NativeR2D2Learner
    _, r2d2 = alp.launch_facts()
    eng = NativeR2D2Learner(batch=1, seq_len=3, burn_in=1, lstm_size=L)
    try:
        _, pf, pb = eng.recurrence_clusters()
    finally:
        eng.close()
    return r2d2(1, 3, 1, 2, L)["R"], pf, pb


def many_chunks_B(L):
    """B with ceil(B / R) > max(P_fwd, P_bwd) and B mod R != 0: the first cluster of each recurrence kernel walks two
    chunks, and the last chunk has R / 2 dead sequences."""
    R, pf, pb = recurrence_plan(L)
    return R * max(pf, pb) + R // 2


def _B(B, L):
    return many_chunks_B(L) if B == MANY else B
APEX_SHAPES = [(B, A) for B in (1, 32, 300) for A in (4, 18)]
APEX_CASES = [("apex", 2, B, A, "init") for B, A in APEX_SHAPES] + \
             [("apex", 2, 32, 18, "trained"), ("apex", 2, 32, 18, "large_returns"), ("apex", 2, 32, 4, "ties"),
              ("apex", 2, 300, 18, "ties"), ("apex", 1, 32, 18, "init"), ("apex", 1, 300, 4, "init")] + \
             [("a3c", 2, B, A, "init") for B, A in APEX_SHAPES] + \
             [("a3c", 2, 32, 18, "trained"), ("a3c", 2, 32, 18, "peaked"), ("a3c", 2, 300, 4, "peaked"),
              ("a3c", 1, 32, 18, "init"), ("a3c", 1, 300, 4, "init")]


def test_case_matrix_reaches_the_edges(native):
    """From the library's own plans, across the matrix: split-K > 1 in heads_l1_fwd, lstm_x_fwd and every conv weight
    gradient (the single-channel conv1 path included) in both math modes, and partial last M tiles (rows not a
    multiple of the 128-row tile) in the forward and the backward of both learners, beside a shape whose tiles are
    all full."""
    apex, r2d2 = alp.launch_facts()
    for mode in (1, 2):
        a = [apex(B, mode) for B in (1, 32, 300)]
        for k in ("heads_l1_fwd", "conv1_wgrad", "conv2_wgrad", "conv3_wgrad"):
            assert max(f[k] for f in a) > 1, (mode, k, a)
        r1 = [r2d2(B, S, C, mode) for B, S, _, _, C in R2D2_SHAPES if C == 1]
        r4 = [r2d2(B, S, C, mode) for B, S, _, _, C in R2D2_SHAPES if C == 4]
        for k in ("lstm_x_fwd", "conv1_wgrad", "conv2_wgrad", "conv3_wgrad"):
            assert max(f[k] for f in r1) > 1 and max(f[k] for f in r4) > 1, (mode, k, r1, r4)
    apex_rows = [2 * B for B, _ in APEX_SHAPES] + [B for B, _ in APEX_SHAPES]
    r2d2_rows = [B * S for B, S, _, _, _ in R2D2_SHAPES]
    assert any(r % alp.TILE for r in apex_rows) and any(r % alp.TILE for r in r2d2_rows)
    assert any(r % alp.TILE == 0 for r in r2d2_rows)              # the benchmark shape: M = 1280, full tiles


@pytest.mark.parametrize("L", WIDTHS)
def test_wide_case_matrix_reaches_the_edges(native, L):
    """At lstm_size 256 and 512, from the library's plan at N = 4L and recurrence_clusters(): split-K > 1 in
    lstm_x_fwd in both math modes, a case with B mod R != 0, a case in which one cluster of the forward and one of the
    BPTT walks two or more chunks of R sequences, and partial last M tiles beside full ones."""
    _, r2d2 = alp.launch_facts()
    R, pf, pb = recurrence_plan(L)
    assert R > 1 and pf >= 1 and pb >= 1, (L, R, pf, pb)
    shapes = [(_B(B, L), S, C) for B, S, _, _, C in WIDE_SHAPES]
    for mode in (1, 2):
        plans = [r2d2(B, S, C, mode, L) for B, S, C in shapes]
        assert all(f["R"] == R for f in plans), (L, plans)
        assert max(f["lstm_x_fwd"] for f in plans) > 1, (L, mode, plans)
    assert any(B % R for B, _, _ in shapes), (L, R, shapes)
    chunks = [-(-B // R) for B, _, _ in shapes]
    assert any(n > pf and n > pb for n in chunks), (L, chunks, pf, pb)
    rows = [B * S for B, S, _ in shapes]
    assert any(r % alp.TILE for r in rows) and any(r % alp.TILE == 0 for r in rows), (L, rows)


def _regime_reached(regime, facts):
    assert facts["finite"], "non-finite output"
    if regime == "trained":
        # every bias has left its zero init and the whole vector moved by >= 0.5 % (L2)
        assert facts["biases_nonzero"] and facts["param_moved_rel_l2"] >= 5e-3, facts
    elif regime == "saturated":
        assert facts["z_abs_gt4"] >= 0.2 and facts["c_abs_max"] > 3, facts
    elif regime == "done_heavy":
        assert 0.2 <= facts["done_rate"] <= 0.45 and facts["done_ends"], facts
    elif regime == "large_returns":
        # Ape-X: the targets; R2D2: the target q that h^-1 reads
        assert facts["target_abs_max"] >= 100, facts
    elif regime == "ties":
        assert facts["tie_rows"] >= 1, facts
    elif regime == "peaked":
        assert 0 < facts["policy_min"] <= 1e-18, facts


def _assert_rows(rows):
    bad = [r for r in rows if not r["ok"]]
    assert not bad, "\n".join("%-22s %-14s err %.3g block %.3g (%s) bar %s%s" % (
        r["kernel"], r["tensor"], r["err"], r["block"], r["where"], r["bar"],
        " bound ratio %.3g" % r["bound_ratio"] if "bound_ratio" in r else "") for r in bad)
    assert np.isfinite([r["err"] for r in rows]).all()


@pytest.mark.parametrize("mode,B,S,bi,A,C,L,regime", R2D2_CASES, ids=[_r2d2_id(c) for c in R2D2_CASES])
def test_r2d2_kernels_against_own_inputs(native, mode, B, S, bi, A, C, L, regime):
    rows, facts = alp.run_r2d2_case(mode, _B(B, L), S, bi, A, C, regime, L=L)
    _regime_reached(regime, facts)
    # at 256 / 512 the o block of dz has its own per-element row
    assert len(rows) == len(alp.R2D2_KERNEL) + 4 + 3 + 6 + 2 + (L != 64)
    _assert_rows(rows)


@pytest.mark.parametrize("L", WIDTHS)
def test_r2d2_td_error_forward_against_own_inputs(native, L):
    """td_error over n = 1 and n = R + 1 sequences (one chunk, and one full chunk plus a chunk of R - 1 dead
    sequences) on one learner: the trunk, zx, the recurrence and its exact state hand-over, q1 and q of each call,
    from the buffers of that call."""
    R = recurrence_plan(L)[0]
    out = alp.run_r2d2_td_error_case(2, (1, R + 1), 15, 7, 4, 1, L)
    assert sorted(out) == [1, R + 1]
    for n, rows in out.items():
        assert len(rows) == len(alp.R2D2_FWD_KERNEL) + 4 + 3, n
        _assert_rows(rows)


@pytest.mark.parametrize("algo,mode,B,A,regime", APEX_CASES)
def test_apex_a3c_kernels_against_own_inputs(native, algo, mode, B, A, regime):
    rows, facts = alp.run_apex_case(algo, mode, B, A, regime)
    _regime_reached(regime, facts)
    assert len(rows) == len(alp.apex_kernels(algo)) + (8 if algo == "apex" else 6)
    _assert_rows(rows)
