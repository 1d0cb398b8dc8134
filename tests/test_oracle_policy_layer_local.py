"""CPU self-check of the per-kernel references of the policy engines' act (tests/policy_layer_parity.py).

  * Fed the float64 oracle's own intermediates (``impala_torch.network``, ``r2d2_torch.network`` / ``Learner.step_q``,
    ``apex_torch.dueling_network``, ``a3c_torch.network``), the references reproduce the oracle's activations, h', c',
    q and policy to 1e-10, the per-split zpart references sum to the oracle's x W, and every check of ``check`` passes:
    a failure of tests/test_gpu_policy_layer_local.py cannot come from a wrong reference.
  * The bounds see small faults: a split-K slab shifted by one K row, an 8-row head block off by 1e-4 whose values are
    small next to the tensor's maximum, and a probability of 1e-12 off by 1 % (which the whole-tensor check passes)."""
import numpy as np
import pytest
import torch

import adam_layer_parity as alp
import policy_layer_parity as plp
from layer_parity import FFMA_DOT
from oracle import a3c_torch as at
from oracle import apex_torch as ax
from oracle import impala_torch as it
from oracle import r2d2_torch as rt

TOL = 1e-10


def _rel(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return float(np.max(np.abs(got - ref))) / max(float(np.max(np.abs(ref))), 1e-300)


def _np(t):
    return t.detach().numpy()


def _oracle_act(family, n, A, C):
    """(buf, out, P, inp, oracle): the buffers and outputs an exact act would produce, from the float64 oracle."""
    P = {k: v.double() for k, v in plp.init_params(family, A, C).items()}
    if family == "impala":
        P["conv3.b"] = P["conv3.b"] - 0.02          # some dead a3 units: the masks matter
    inp = plp.make_inputs(family, n, A, C)
    x = torch.from_numpy(alp._frames(inp["state"]))
    pa = torch.from_numpy(inp["pa"].astype(np.int64))
    acts = torch.arange(A)
    buf = {"e1": _np(torch.relu(torch.nn.functional.one_hot(acts, A).double() @ P["emb1.w"] + P["emb1.b"])),
           "table": _np(it.action_embedding(P, acts, A))}
    out, orc = {}, {}
    if family in ("impala", "r2d2"):
        h0, c0 = torch.from_numpy(inp["h"]).double(), torch.from_numpy(inp["c"]).double()
    if family == "impala":
        actor, _, c, h, taps = it.network(P, x, pa, h0, c0, A, 256, return_taps=True)
        out.update(policy=_np(actor), h=_np(h), c=_np(c))
        xw = torch.cat([taps["a3"].reshape(n, -1), taps["emb"], h0], 1) @ P["lstm.w"]
    elif family == "r2d2":
        q, h, c, taps = rt.network(P, x, pa, h0, c0, A)
        out.update(q=_np(q), h=_np(h), c=_np(c))
        emb = it.action_embedding(P, pa, A)
        xw = torch.cat([taps["a3"].reshape(n, -1), emb, h0], 1) @ P["lstm.w"]
        L = rt.Learner({k: v.float() for k, v in P.items()}, None, torch.float64, num_action=A, input_shape=(84, 84, C))
        orc["step_q"] = L.step_q(inp["state"], inp["h"], inp["c"], inp["pa"])
    elif family == "apex":
        q, taps = ax.dueling_network(P, x, pa, A, return_taps=True)
        out["q"] = _np(q)
        xw = torch.cat([taps["a3"].reshape(n, -1), taps["emb"]], 1) @ torch.cat([P["value1.w"], P["mean1.w"]], 1)
    else:
        actor, _, taps = at.network(P, x, pa, A, return_taps=True)
        out["policy"] = _np(actor)
        xw = torch.cat([taps["a3"].reshape(n, -1), it.action_embedding(P, pa, A)], 1) @ P["actor1.w"]
    buf.update(a1=_np(taps["a1"]), a2=_np(taps["a2"]), a3=_np(taps["a3"]).reshape(n, -1))
    W = {k: _np(v) for k, v in P.items()}
    xk = plp.skinny_x(buf["a3"], buf["table"], inp["pa"], inp.get("h"))
    buf["zpart"], _ = plp.skinny_references(xk, plp.first_weight(family, W), plp.SPLITS[family])
    out["action"] = plp.expected_actions(family, out, inp)
    idx = np.arange(n), out["action"]
    if family == "a3c":
        out["max_prob"] = out["policy"][idx]
    elif family in ("r2d2", "apex"):
        out["q_action"] = out["q"][idx]
    orc.update(out)
    orc["xW"] = _np(xw)
    return buf, out, P, inp, orc


CASES = [("impala", 9, 18, 4), ("impala", 3, 2, 4), ("r2d2", 9, 4, 1), ("r2d2", 5, 32, 4), ("apex", 9, 4, 4),
         ("apex", 3, 32, 4), ("a3c", 9, 18, 4), ("a3c", 3, 2, 4)]


@pytest.mark.parametrize("family,n,A,C", CASES)
def test_references_reproduce_the_oracle(family, n, A, C):
    buf, out, P, inp, orc = _oracle_act(family, n, A, C)
    rows, ref = plp.check(family, buf, out, P, inp, A)
    errs = {k: _rel(ref[k], buf[k]) for k in ("a1", "a2", "a3", "e1", "table")}
    errs["sum zpart = xW"] = _rel(ref["zpart"].sum(0), orc["xW"])
    if family in ("impala", "r2d2"):
        errs.update(h=_rel(ref["h"], orc["h"]), c=_rel(ref["c"], orc["c"]))
    if family in ("impala", "a3c"):
        errs["policy"] = _rel(ref["policy"], orc["policy"])
    else:
        errs["q"] = _rel(ref["q"], orc["q"])
    if family == "r2d2":
        q, h, c = orc["step_q"]
        errs.update(step_q=_rel(ref["q"], q), step_h=_rel(ref["h"], h), step_c=_rel(ref["c"], c))
    assert all(v < TOL for v in errs.values()), errs
    bad = [r for r in rows if not r["ok"]]
    assert not bad, bad
    assert len(rows) == {"impala": 11, "r2d2": 11, "apex": 9, "a3c": 10}[family]


def test_row_tiles_and_straddling_splits():
    assert sorted({plp.row_tile(n) for n in plp.ROWS}) == [8, 16, 32, 64]
    assert [plp.row_tile(n) for n in (8, 9, 16, 17, 32, 33)] == [8, 16, 16, 32, 32, 64]
    assert {f: plp.split_k(f) for f in plp.FAMILIES} == dict(impala=228, r2d2=72, apex=64, a3c=64)
    assert {f: plp.straddling_splits(f) for f in plp.FAMILIES} == dict(impala=[13, 14], r2d2=[43, 47], apex=[], a3c=[])


def _skinny_case():
    """A [9, 3648] x [3648, 1024] case from the oracle's IMPALA intermediates (float32 values)."""
    buf, out, P, inp, _ = _oracle_act("impala", 9, 18, 4)
    x = plp.skinny_x(buf["a3"], buf["table"], inp["pa"], inp["h"]).astype(np.float32)
    W = P["lstm.w"].numpy().astype(np.float32)
    return x, W


def test_splitk_bound_holds_for_float32_and_sees_a_shifted_slab():
    x, W = _skinny_case()
    S = plp.SPLITS["impala"]
    kK = plp.split_k("impala")
    ref, bound = plp.skinny_references(x.astype(np.float64), W.astype(np.float64), S)
    got = np.stack([x[:, s * kK:(s + 1) * kK] @ W[s * kK:(s + 1) * kK] for s in range(S)]).astype(np.float64)
    r = plp.splitk_row("skinny_splitk_fwd", got, ref, bound)
    assert r["ok"] and 0 < r["bound_ratio"] < 1, r
    for s in plp.straddling_splits("impala") + [0, S - 1]:
        bad = got.copy()
        lo = s * kK
        w = W[lo + 1:lo + kK + 1] if s < S - 1 else W[lo - 1:lo + kK - 1]      # the slab one K row off
        bad[s] = (x[:, lo:lo + kK] @ w).astype(np.float64)
        r = plp.splitk_row("skinny_splitk_fwd", bad, ref, bound)
        assert not r["ok"] and r["where"].startswith("split %d " % s), (s, r)


def test_head_block_error_is_seen_per_cta():
    rng = np.random.RandomState(3)
    ref = rng.standard_normal((24, 6))
    ref[8:16] *= 1e-2                                   # one head CTA whose values are small next to the maximum
    got = ref.copy()
    got[8:16] *= 1 + 1e-4
    assert plp.head_row("k", "q", ref, ref, 8)["ok"]
    r = plp.head_row("k", "q", got, ref, 8)
    assert not r["ok"] and r["where"] == "cta1" and r["err"] <= FFMA_DOT, r


def test_log_space_sees_a_small_probability_the_tensor_check_misses():
    logits = np.log(np.array([[0.5, 0.3, 0.2 - 1e-12, 1e-12], [0.25, 0.25, 0.25, 0.25]]))
    p = np.exp(plp.log_softmax(logits))
    assert abs(p[0, 3] - 1e-12) < 1e-20
    p32 = p.astype(np.float32).astype(np.float64)
    assert plp.log_space_row("k", p32, logits, 8)["ok"]
    bad = p32.copy()
    bad[0, 3] *= 1.01
    assert plp.head_row("k", "policy", bad, p, 8)["ok"]       # the whole-tensor and block bars pass it
    r = plp.log_space_row("k", bad, logits, 8)
    assert not r["ok"] and r["where"] == "cta 0 row 0 action 3", r
    zero = p32.copy()
    zero[0, 3] = 0.0                                          # a probability flushed to zero
    assert not plp.log_space_row("k", zero, logits, 8)["ok"]
