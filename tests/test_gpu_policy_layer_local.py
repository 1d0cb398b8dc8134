"""-m gpu: every kernel of the IMPALA, R2D2, Ape-X and A3C policy engines' act checked on its own, against a float64
reference computed from the buffers that kernel read in the same act (tests/policy_layer_parity.py; its references are
checked against the float64 oracle by tests/test_oracle_policy_layer_local.py).  The conv trunk and the embedding are
held to the learners' bars, the split-K partials of the skinny GEMM per element to the deterministic bound of a float32
FFMA chain (the report names the split, the 128-column chunk and the row), h' and c' per element to
layer_parity.lstm_bounds, q and policy per tensor and per head CTA, the softmax in log space, the action rule exactly.

Case matrix (one engine per family, A and C, max_batch 64, CUDA graphs on):
  * n in {1, 8, 9, 16, 17, 32, 33, 64}: every row tile R = 8 / 16 / 32 / 64 of the skinny GEMM and both sides of each
    boundary, and partial 8-row head CTAs; IMPALA and A3C at A in {2, 18, 32}, Ape-X at A in {4, 32}, R2D2 at A in
    {4, 32} and C in {1, 4};
  * regimes at n in {9, 64}: trained (the family's learner at a raised learning rate, then sync_from), saturated LSTM
    gates (IMPALA, R2D2), a peaked softmax with min p <= 1e-18 (IMPALA, A3C) and IMPALA's fp16-split conv1 at
    |w| ~ 1e-4 and ~ 5.  Every case asserts that it reached its regime;
  * row independence, bitwise: the rows of a 64-row act against the same rows of acts on its prefixes and on a shifted
    17-row window.  Every output element is one fixed-order chain that depends neither on the row tile nor on where the
    row sits in it, so no tolerance is needed."""
import numpy as np
import pytest

import policy_layer_parity as plp

pytestmark = pytest.mark.gpu

INIT_CASES = ([("impala", n, A, 4) for A in (2, 18, 32) for n in plp.ROWS] +
              [("a3c", n, A, 4) for A in (2, 18, 32) for n in plp.ROWS] +
              [("apex", n, A, 4) for A in (4, 32) for n in plp.ROWS] +
              [("r2d2", n, A, C) for C in (1, 4) for A in (4, 32) for n in plp.ROWS])
REGIME_CASES = [(f, n, A, C, r)
                for f, A, C, regimes in (("impala", 18, 4, ("trained", "saturated", "peaked", "conv1_w_1e-4",
                                                            "conv1_w_5")),
                                         ("r2d2", 4, 1, ("trained", "saturated")),
                                         ("apex", 4, 4, ("trained",)),
                                         ("a3c", 18, 4, ("trained", "peaked")))
                for r in regimes for n in (9, 64)]
ROWS_CHECKED = dict(impala=11, r2d2=11, apex=9, a3c=10)


@pytest.fixture(scope="module")
def engines(native):
    """engines(family, A, C): one engine per configuration for the whole module."""
    if native.device_count() < 1:
        pytest.skip("needs a CUDA device")
    cache = {}

    def get(family, A, C):
        if (family, A, C) not in cache:
            cache[family, A, C] = plp.make_engine(family, A, C)
        return cache[family, A, C]
    yield get
    for p in cache.values():
        p.close()


def test_case_matrix_reaches_the_edges():
    """Every family's rows reach all four row tiles of launch_skinny_splitk, both sides of each tile boundary and a
    partial 8-row head CTA beside full ones; the straddling splits (a part boundary of x inside the split) are the
    ones the per-split check names."""
    for family in plp.FAMILIES:
        ns = sorted({c[1] for c in INIT_CASES if c[0] == family})
        assert sorted({plp.row_tile(n) for n in ns}) == [8, 16, 32, 64], (family, ns)
        for r in (8, 16, 32):
            assert r in ns and r + 1 in ns and plp.row_tile(r) != plp.row_tile(r + 1), (family, r)
        assert any(n % 8 and n > 8 for n in ns) and any(n % 8 == 0 for n in ns), family
    assert plp.straddling_splits("impala") == [13, 14] and plp.straddling_splits("r2d2") == [43, 47]
    assert plp.straddling_splits("apex") == plp.straddling_splits("a3c") == []


@pytest.mark.parametrize("family", plp.FAMILIES)
def test_read_hook(native, family):
    """The read hook before and after an act, its dims, and its refusals (a wrong count, an unknown name)."""
    if native.device_count() < 1:
        pytest.skip("needs a CUDA device")
    A, C = 4, 1
    pol = plp.make_engine(family, A, C, max_batch=9)
    try:
        fn = getattr(native.lib, "drl_%s_read_buffer" % pol.prefix)
        a = np.empty(5 * 3136, np.float32)
        assert pol.buffer_dims() == (0, plp.SPLITS[family], plp.COLS[family])
        assert fn(pol._h, b"a3", native.ptr(a), a.size) == native.DRL_ERR_STATE
        pol.set_params(plp.flatten(family, plp.init_params(family, A, C)))
        plp.act(pol, family, plp.make_inputs(family, 5, A, C))
        assert pol.buffer_dims() == (5, plp.SPLITS[family], plp.COLS[family])
        assert fn(pol._h, b"a3", native.ptr(a), a.size) == native.DRL_OK
        assert fn(pol._h, b"a3", native.ptr(a), a.size - 1) == native.DRL_ERR_INVALID
        assert fn(pol._h, b"a4", native.ptr(a), a.size) == native.DRL_ERR_INVALID
        assert np.array_equal(pol.read_buffer("a3").ravel(), a)
        assert pol.read_buffer("zpart").shape == (plp.SPLITS[family], 5, plp.COLS[family])
    finally:
        pol.close()


def _assert_rows(rows):
    bad = [r for r in rows if not r["ok"]]
    assert not bad, "\n".join("%-28s %-10s err %.3g block %.3g (%s) bar %s%s" % (
        r["kernel"], r["tensor"], r["err"], r["block"], r["where"], r["bar"],
        " bound ratio %.3g" % r["bound_ratio"] if "bound_ratio" in r else "") for r in bad)


def _case(engines, family, n, A, C, regime):
    rows, facts = plp.run_case(family, n, A, C, regime, pol=engines(family, A, C))
    assert facts["finite"], "non-finite output"
    assert facts["buffer_dims"] == (n, plp.SPLITS[family], plp.COLS[family]), facts
    assert len(rows) == ROWS_CHECKED[family]
    return rows, facts


@pytest.mark.parametrize("family,n,A,C", INIT_CASES)
def test_policy_kernels_against_own_inputs(engines, family, n, A, C):
    rows, _ = _case(engines, family, n, A, C, "init")
    _assert_rows(rows)


@pytest.mark.parametrize("family,n,A,C,regime", REGIME_CASES)
def test_policy_kernels_in_regime(engines, family, n, A, C, regime):
    rows, facts = _case(engines, family, n, A, C, regime)
    if regime == "trained":
        # every bias has left its init and the whole vector moved by >= 0.5 % (L2)
        assert facts["biases_nonzero"] and facts["param_moved_rel_l2"] >= 5e-3, facts
    elif regime == "saturated":
        assert facts["z_abs_gt4"] >= 0.2, facts
    elif regime == "peaked":
        assert 0 < facts["policy_ref_min"] <= 1e-18, facts
    elif regime.startswith("conv1_w_"):
        target = float(regime[len("conv1_w_"):])
        assert 0.5 * target <= facts["conv1_w_median_abs"] <= 2 * target, facts
    _assert_rows(rows)


@pytest.mark.parametrize("family,A,C", [("impala", 18, 4), ("r2d2", 4, 1), ("r2d2", 32, 4), ("apex", 4, 4),
                                        ("a3c", 18, 4)])
def test_rows_do_not_depend_on_the_other_rows(engines, family, A, C):
    diffs = plp.row_independence(engines(family, A, C), family, A, C)
    assert len(diffs) == 5 * (len(plp.BUFFERS) + {"impala": 4, "r2d2": 5, "apex": 3, "a3c": 3}[family])
    bad = {k: v for k, v in diffs.items() if v}
    assert not bad, bad
