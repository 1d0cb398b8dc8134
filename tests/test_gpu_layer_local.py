"""-m gpu: every kernel of the IMPALA learner step checked on its own, against a float64 reference computed from the
buffers that kernel read in the same step (tests/layer_parity.py; its references are checked against the float64 oracle
by tests/test_oracle_layer_local.py).  The bars come from each core's error model (layer_parity.bars), per tensor and per
block; the conv1 forward of math mode 5 is held to the per-element bound of its fp16 split (layer_parity.conv1_bound),
the LSTM gates, c1 and h1 to the per-element bounds of the lstm_fwd error model (layer_parity.lstm_bounds).

Case matrix: math mode 5 at four shapes in five parameter regimes (glorot init; scaled: saturated LSTM gates and a
mostly dead conv3; trained: 20 steps at a raised learning rate, checked on a fresh batch; conv1.w at a typical |w| of
1e-4 and of 5), math modes 1, 2 and 3 at two shapes from init.  Every case asserts that it reached what it claims."""
import numpy as np
import pytest

import layer_parity as lp

pytestmark = pytest.mark.gpu

SHAPES = [(32, 20, 18),    # the benchmark shape
          (1, 3, 2),       # Mb = 1, three frames: partial tiles everywhere
          (5, 32, 32),     # the largest A, odd sizes
          (128, 20, 18)]   # many frames per persistent conv1 CTA, multi-split weight gradients
CASES = [(5, B, T, A, r) for (B, T, A) in SHAPES for r in lp.REGIMES] + \
        [(m, B, T, A, "init") for m in (1, 2, 3) for (B, T, A) in (SHAPES[0], SHAPES[2])]


def test_case_matrix_reaches_the_edges(native):
    """Across the math-mode-5 shapes: partial last M tiles, split-K > 1 in every conv weight gradient, and more than two
    frames per persistent conv1 CTA (the double-buffered frame barriers wrap their phase) in both conv1 kernels."""
    facts = [lp.launch_facts(B, T) for B, T, _ in SHAPES]
    partial = set().union(*[f["partial_tiles"] for f in facts])
    assert {"lstm_fwd/heads_fwd", "heads_dgrad/lstm_dgrad", "conv2_fwd", "conv3_fwd", "conv3_dgrad",
            "conv2_dgrad"} <= partial, partial
    assert any(f["partial_tiles"] == [] for f in facts)           # and a shape whose tiles are all full
    for k in ("conv1_wgrad", "conv2_wgrad", "conv3_wgrad"):
        assert max(f["splits"][k] for f in facts) > 1, k
    assert max(f["conv1_fwd_frames_per_cta"] for f in facts) > 2
    assert max(f["conv1_wgrad_frames_per_cta"] for f in facts) > 2
    assert min(f["conv1_fwd_frames_per_cta"] for f in facts) == 1


def _regime_reached(regime, facts):
    assert facts["finite"], "non-finite output"
    if regime == "scaled":
        assert facts["z_abs_gt4"] >= 0.2, facts
        assert facts["a3_zero"] >= 0.5, facts
    elif regime == "trained":
        # every bias has left its zero init; the whole vector moved by >= 0.5 % (L2; 8 % at the benchmark shape, 0.9 %
        # at B = 1, T = 3, whose single backward row gives the smallest gradients)
        assert facts["biases_nonzero"] and facts["param_moved_rel_l2"] >= 5e-3, facts
    elif regime == "conv1_w_1e-4":
        assert 0.5e-4 <= facts["conv1_w_median_abs"] <= 2e-4, facts
    elif regime == "conv1_w_5":
        assert 2.5 <= facts["conv1_w_median_abs"] <= 10, facts


@pytest.mark.parametrize("mode,B,T,A,regime", CASES)
def test_kernels_against_own_inputs(native, mode, B, T, A, regime):
    rows, facts = lp.run_case(mode, B, T, A, regime)
    _regime_reached(regime, facts)
    assert len(rows) == len(lp.KERNEL)
    bad = [r for r in rows if not r["ok"]]
    assert not bad, "\n".join("%-22s %-10s err %.3g block %.3g (%s) bar %s%s" % (
        r["kernel"], r["tensor"], r["err"], r["block"], r["where"], r["bar"],
        " bound ratio %.3g" % r["bound_ratio"] if "bound_ratio" in r else "") for r in bad)
    assert np.isfinite([r["err"] for r in rows]).all()
