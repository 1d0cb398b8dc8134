"""-m gpu: every kernel of the Ape-X, A3C and R2D2 learner steps checked on its own, against a float64 reference
computed from the buffers that kernel read in the same step (tests/adam_layer_parity.py; its references are checked
against the float64 oracle by tests/test_oracle_adam_layer_local.py).  Same metric, per-block reporting and failure
message as tests/test_gpu_layer_local.py; the R2D2 recurrence is held per element to layer_parity.lstm_bounds with the
K = 64 FFMA dot product as the pre-activation bar, the loss kernels per element to the rounding bounds of the values
they combine, and the recurrence's state hand-over and the gradient rows outside the loss window bitwise.

Case matrix, math mode 2 (3xTF32, the default) unless noted:
  * R2D2 (B, S, burn_in, A, C) from init at the reference config, the benchmark shape (Nt = 39 > 32: the TD kernel's
    lane loop; B > 8: its warp loop), M = 2 (partial tiles everywhere), A = 32 and B = 140 (more recurrence CTAs than
    SMs); trained, done-heavy, large-return and exact next-q tie steps at the reference config; saturated gates at
    the benchmark shape;
    math mode 1 at the reference config and the benchmark shape.
  * Ape-X and A3C at B = 1, 32 and 300 (n > 256: the loss kernels' block-stride loop) with A = 4 and 18 from init;
    trained, large returns (Ape-X, reward_clipping "none"), exact next-q ties (Ape-X) and a peaked policy (A3C);
    math mode 1 at two shapes.
Every case asserts that it reached its regime."""
import numpy as np
import pytest

import adam_layer_parity as alp

pytestmark = pytest.mark.gpu

R2D2_SHAPES = [(16, 15, 7, 4, 1),     # the reference config
               (16, 80, 40, 4, 1),    # the benchmark shape
               (1, 2, 0, 2, 4),       # M = 2
               (5, 7, 5, 32, 4),      # A = 32
               (140, 4, 1, 4, 1)]     # more sequences than SMs
R2D2_CASES = [(2,) + s + ("init",) for s in R2D2_SHAPES] + \
             [(2,) + R2D2_SHAPES[0] + (r,) for r in ("trained", "done_heavy", "large_returns", "ties")] + \
             [(2,) + R2D2_SHAPES[1] + ("saturated",)] + \
             [(1,) + s + ("init",) for s in R2D2_SHAPES[:2]]
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


@pytest.mark.parametrize("mode,B,S,bi,A,C,regime", R2D2_CASES)
def test_r2d2_kernels_against_own_inputs(native, mode, B, S, bi, A, C, regime):
    rows, facts = alp.run_r2d2_case(mode, B, S, bi, A, C, regime)
    _regime_reached(regime, facts)
    assert len(rows) == len(alp.R2D2_KERNEL) + 4 + 3 + 6 + 2
    _assert_rows(rows)


@pytest.mark.parametrize("algo,mode,B,A,regime", APEX_CASES)
def test_apex_a3c_kernels_against_own_inputs(native, algo, mode, B, A, regime):
    rows, facts = alp.run_apex_case(algo, mode, B, A, regime)
    _regime_reached(regime, facts)
    assert len(rows) == len(alp.apex_kernels(algo)) + (8 if algo == "apex" else 6)
    _assert_rows(rows)
