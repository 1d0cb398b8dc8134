"""CPU self-check of the per-kernel references of the Ape-X, A3C and R2D2 steps (tests/adam_layer_parity.py): fed the
float64 oracle's own intermediates in device row order, every reference reproduces the oracle's activations, its q
values / policy / losses, its activation gradients and every parameter gradient to 1e-10.  A failure of
tests/test_gpu_adam_layer_local.py therefore cannot come from a wrong reference."""
import numpy as np
import pytest
import torch

import adam_layer_parity as alp
import layer_parity as lp
import parity
import r2d2_parity
from oracle import a3c_torch as at
from oracle import apex_torch as ax
from oracle import r2d2_torch as rt

TOL = 1e-10
CONV = (("a1", (20, 20, 32)), ("a2", (9, 9, 64)), ("a3", (7, 7, 64)))


def _params(p, seed=7):
    """the given glorot kernels with small non-zero biases (every bias path is exercised)."""
    g = torch.Generator().manual_seed(seed)
    for k in p:
        if k.endswith(".b"):
            p[k] = (torch.rand(p[k].shape, generator=g, dtype=torch.float64) - 0.5) * 0.1
    return p


def _np(t):
    return t.detach().numpy()


def _act_grads(loss, params, acts):
    """d loss / d params (by name) and d loss / d each tensor of ``acts``."""
    names = list(params)
    g = torch.autograd.grad(loss, [params[n] for n in names] + list(acts), allow_unused=True)
    pg = {n: (_np(x) if x is not None else np.zeros(tuple(params[n].shape))) for n, x in zip(names, g)}
    return pg, [_np(x) for x in g[len(names):]]


def _converge(step, buf, passes):
    """Run ``step(buf)`` (which rewrites the derived buffers from the references) ``passes`` times: a fixed point once
    ``passes`` exceeds the depth of the dependency chain."""
    for _ in range(passes):
        step(buf)


def _bad(errs):
    return {k: v for k, v in errs.items() if not v < TOL}


# ------------------------------------------------------------------------------------------------------------------
# Ape-X / A3C
# ------------------------------------------------------------------------------------------------------------------
def _apex_case(algo, clip, B=3, A=5):
    mod = ax if algo == "apex" else at
    batch = ax.make_transitions(B, A=A, seed=11 + B)
    batch["reward"] = (batch["reward"] * 3).astype(np.float32)       # both sides of the clipping
    batch["done"][0] = True
    params = _params(mod.init_params(0, torch.float64, num_action=A))
    sv, sm = alp.stream_names(algo)
    img = lambda s: torch.from_numpy((np.asarray(s).astype(np.float64) / 255).astype(np.float32)).to(torch.float64)
    a = torch.from_numpy(batch["action"].astype(np.int64))
    if algo == "apex":
        target = ax.init_params(1, torch.float64, num_action=A)
        L = ax.Learner(params, target, torch.float64, num_action=A, reward_clipping=clip)
        o = L.losses(*[batch[k] for k in ax.TRAIN_FIELDS[:-1]], is_weight=batch["is_weight"])
        loss = o["value_loss"]
        P = L.params
        _, nt = ax.dueling_network(L.params, img(batch["next_state"]), a, A, return_taps=True)
    else:
        cfg = dict(num_action=A, reward_clipping=clip)
        L = at.Learner(params, torch.float64, **cfg)
        o = L.losses(*[batch[k] for k in at.TRAIN_FIELDS])
        loss = o["total_loss"]
        P = L.params
        _, _, nt = at.network(L.params, img(batch["next_state"]), a, A, return_taps=True)
    tp = o["taps"]
    grads, ag = _act_grads(loss, P, [tp[k] for k, _ in CONV])
    buf = {}
    for (k, shp), g in zip(CONV, ag):
        both = np.concatenate([_np(tp[k]), _np(nt[k])]).reshape((2 * B,) + shp)
        buf[k] = both.reshape(2 * B, -1) if k == "a3" else both
        d = g.reshape((B,) + shp) * (both[:B] > 0)
        buf["d" + k] = d.reshape(B, -1) if k == "a3" else d
    shapes = {"e1": (A, 256), "emb": (A, 256), "hid1": (2, 2 * B, 256), "hid2": (2, 2 * B, 256),
              "vstream": (2 * B, A), "mstream": (2 * B,), "policy": (2 * B, A), "dq": (B, 32), "dmean": (B, 32),
              "dhid2": (2, B, 256), "dhid1": (2, B, 256), "du": (B, 256)}
    buf.update({k: np.zeros(s) for k, s in shapes.items()})
    gamma = L.cfg["discount_factor"]
    state = {}

    def step(b):
        ref = alp.apex_references(b, P, batch, B, A, algo)
        for k in ("e1", "emb", "hid1", "hid2", "vstream", "mstream", "policy", "dhid2", "dhid1", "du"):
            b[k] = ref[k]
        if algo == "apex":
            v, m = b["vstream"], b["mstream"]
            td = alp.apex_td(v[:B] - m[:B, None], v[B:] - m[B:, None], _np(o["target_q"]), batch, gamma,
                             clip == "abs_one", A)
        else:
            td = alp.a3c_loss(b["policy"][:B], b["mstream"][:B], b["mstream"][B:], batch,
                              dict(at.DEFAULT_CFG, reward_clipping=clip))
        b["dq"][:, :A], b["dmean"][:, 0] = td["dq"], td["dmean"]
        state.update(ref=ref, td=td)
    _converge(step, buf, 12)
    ref, td = state["ref"], state["td"]
    errs = {}
    for k, _ in CONV:
        errs[k] = parity.rel_err(ref[k], buf[k])
    for k in ("da3", "da2", "da1"):
        errs[k] = parity.rel_err(ref[k], buf[k])
    for n in grads:
        errs["grad/" + n] = parity.rel_err(ref[n], grads[n])
    assert len([k for k in errs if k.startswith("grad/")]) == 22
    if algo == "apex":
        errs["main_q"] = parity.rel_err(buf["vstream"][:B] - buf["mstream"][:B, None], _np(o["main_q"]))
        errs["next_main_q"] = parity.rel_err(buf["vstream"][B:] - buf["mstream"][B:, None], _np(o["next_main_q"]))
        errs["value"] = parity.rel_err(buf["vstream"][:B], _np(tp["value"]))
        for k, ok in (("target_value", "target_value"), ("sav", "state_action_value")):
            errs[k] = parity.rel_err(td[k], _np(o[ok]))
        errs["loss"] = parity.rel_err(td["loss"], float(o["value_loss"].detach()))
    else:
        errs["policy"] = parity.rel_err(buf["policy"][:B], _np(o["policy"]))
        errs["value"] = parity.rel_err(buf["mstream"][:B], _np(o["value"]))
        errs["next_value"] = parity.rel_err(buf["mstream"][B:], _np(o["next_value"]))
        errs["adv"] = parity.rel_err(td["adv"], _np(o["advantage"]))
        for k in ("pi_loss", "baseline_loss", "entropy"):
            errs[k] = parity.rel_err(td[k], float(o[k].detach()))
    assert all(np.abs(buf[k]).max() > 0 for k in shapes), "a derived buffer is all zero"
    return errs


@pytest.mark.parametrize("clip", ["abs_one", "none"])
def test_apex_references_reproduce_oracle(clip):
    bad = _bad(_apex_case("apex", clip))
    assert not bad, bad


@pytest.mark.parametrize("clip", ["abs_one", "soft_asymmetric"])
def test_a3c_references_reproduce_oracle(clip):
    bad = _bad(_apex_case("a3c", clip))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------------------------
# R2D2
# ------------------------------------------------------------------------------------------------------------------
def _r2d2_fixed_point(L, B, S, bi, A, C, seed, dones):
    """The R2D2 step's buffers as an exact (float64) device would leave them at width L: the oracle's conv activations
    and gradients, q and TD gradients, and every LSTM / head buffer iterated to the fixed point of the references.
    ``dones``: the (sequence, step) pairs that end an episode.  -> dict(buf, grads, ref, td, taps, out, batch, params,
    inp, o)."""
    kw = dict(num_action=A, lstm_size=L, input_shape=(84, 84, C))
    batch = r2d2_parity.make_batch(B, S, A, C, seed, L=L)
    batch["done"][:] = False
    for b, t in dones:
        batch["done"][b, t] = True
    params = _params(rt.init_params(0, torch.float64, **kw))
    target = rt.init_params(1, torch.float64, **kw)
    Lr = rt.Learner(params, target, torch.float64, seq_len=S, burn_in=bi, **kw)
    o = Lr.losses(*[batch[k] for k in rt.TRAIN_FIELDS[:-1]], weight=batch["weight"])
    taps = o["taps"]
    acts = [taps[t][k] for t in range(S) for k, _ in CONV]
    grads, ag = _act_grads(o["value_loss"], Lr.params, acts)
    M = B * S
    buf = {}
    for ci, (k, shp) in enumerate(CONV):
        a = np.stack([_np(taps[t][k]) for t in range(S)]).reshape((M,) + shp)        # time-major
        d = np.stack([ag[t * len(CONV) + ci] for t in range(S)]).reshape((M,) + shp) * (a > 0)
        buf[k], buf["d" + k] = (a.reshape(M, -1), d.reshape(M, -1)) if k == "a3" else (a, d)
    mq, tq = _np(o["main_q"]), _np(o["target_q"])
    buf["q"] = lp.time_major(mq)
    shapes = {"e1": (A, 256), "emb": (A, 256), "zx": (M, 4 * L), "gates": (M, 4 * L), "tc": (M, L), "hout": (M, L),
              "q1": (M, 128), "dq1": (M, 128), "dhout": (M, L), "dz": (M, 4 * L), "du": (M, 256)}
    buf.update({k: np.zeros(s) for k, s in shapes.items()})
    inp = alp.r2d2_inputs(batch)
    keep = (~inp["done"]).astype(np.float64).T.reshape(M, 1)
    buf["hin"] = np.concatenate([inp["h0"], np.zeros((M - B, L))])
    buf["cin"] = np.concatenate([inp["c0"], np.zeros((M - B, L))])
    td = alp.r2d2_td(mq, tq, batch, bi, Lr.cfg["discount_factor"], B, S, A)
    buf["dq"], buf["dmean"] = np.zeros((M, 32)), np.zeros((M, 32))
    buf["dq"][:, :A], buf["dmean"][:, 0] = td["dq"], td["dmean"]
    state = {}

    def step(b):
        ref = alp.r2d2_references(b, Lr.params, batch, B, S, A, L)
        for k in shapes:
            b[k] = ref[k]
        b["hin"] = np.concatenate([inp["h0"], (ref["hout"] * keep)[:M - B]])
        b["cin"] = np.concatenate([inp["c0"], ref["cnext"]])
        state["ref"] = ref
    _converge(step, buf, 2 * S + 10)
    taps_out = dict(main_q=mq, target_q=tq, target_value=_np(o["target_value"]),
                    state_action_value=_np(o["state_action_value"]))
    out = dict(loss=float(o["value_loss"].detach()), td=td["td"])
    return dict(buf=buf, grads=grads, ref=state["ref"], td=td, taps=taps_out, out=out, batch=batch, params=Lr.params,
                inp=inp, o=o, shapes=shapes, cfg=Lr.cfg)


def test_r2d2_references_reproduce_oracle():
    """Dones in mid-sequence (the carry is cut inside the window and inside the burn-in) and burn-in > 0."""
    _references_reproduce_oracle(64)


@pytest.mark.parametrize("L", [256, 512])
def test_r2d2_references_reproduce_oracle_at_width(L):
    """As test_r2d2_references_reproduce_oracle, at lstm_size 256 and 512 (the cluster recurrence's widths)."""
    _references_reproduce_oracle(L)


def _references_reproduce_oracle(L):
    B, S, bi, A, C = 2, 6, 2, 3, 1
    fx = _r2d2_fixed_point(L, B, S, bi, A, C, 31, [(0, 1), (1, 3)])
    ref, buf, td, o, grads, inp = fx["ref"], fx["buf"], fx["td"], fx["o"], fx["grads"], fx["inp"]
    errs = {}
    for k, _ in CONV:
        errs[k] = parity.rel_err(ref[k], buf[k])
    for k in ("da3", "da2", "da1"):
        errs[k] = parity.rel_err(ref[k], buf[k])
    errs["q"] = parity.rel_err(ref["q"], buf["q"])
    errs["gates"] = parity.rel_err(ref["gates"], alp._gates(ref["z"], L))
    errs["tc"] = parity.rel_err(ref["tc"], np.tanh(ref["c"]))
    for k, ok in (("target_value", "target_value"), ("sav", "state_action_value")):
        errs[k] = parity.rel_err(td[k], _np(o[ok]))
    errs["loss"] = parity.rel_err(td["loss"], float(o["value_loss"].detach()))
    for n in grads:
        errs["grad/" + n] = parity.rel_err(ref[n], grads[n])
    assert len([k for k in errs if k.startswith("grad/")]) == 18
    assert all(np.abs(buf[k]).max() > 0 for k in fx["shapes"]), "a derived buffer is all zero"
    # the window, the burn-in and the cut carry are all exercised
    assert np.abs(td["dq"]).max() > 0 and inp["done"][:, :S - 1].any() and bi > 0
    bad = _bad(errs)
    assert not bad, bad


# ------------------------------------------------------------------------------------------------------------------
# R2D2 at lstm_size 256 / 512: each bug of the cluster recurrence or of a wide GEMM fails its kernel's row by >= 10x
# ------------------------------------------------------------------------------------------------------------------
MUT_S, MUT_BI, MUT_A = 4, 1, 3
MUT_B = {256: 10, 512: 2}           # at 256: two chunks of R = 8 sequences, the second one partial
MUT_R = 8                           # sequences per cluster pass at 256 (R2Clu<256>::R)


@pytest.fixture(scope="module")
def r2d2_wide():
    """The oracle-consistent R2D2 buffers at 256 (dones in sequences 0 and 3) and at 512, built once: {L: fixture}."""
    return {256: _r2d2_fixed_point(256, MUT_B[256], MUT_S, MUT_BI, MUT_A, 1, 57, [(0, 1), (3, 2)]),
            512: _r2d2_fixed_point(512, MUT_B[512], MUT_S, MUT_BI, MUT_A, 1, 57, [(0, 1)])}


def _rows(fx, L, buf=None, grads=None):
    rows, _ = alp.check_r2d2(fx["buf"] if buf is None else buf, fx["grads"] if grads is None else grads, fx["params"],
                             fx["batch"], fx["taps"], fx["out"], MUT_B[L], MUT_S, MUT_BI, MUT_A,
                             fx["cfg"]["discount_factor"], L)
    return rows


def _excess(row):
    """How far a row misses: its bound ratio, its error over its bar, or (exact rows) inf when any element differs."""
    if "bound_ratio" in row:
        return row["bound_ratio"]
    if row["bar"] == "exact":
        return float("inf") if row["err"] > 0 else 0.0
    return max(row["err"], row["block"]) / row["bar"]


def _W(fx):
    return _np(fx["params"]["lstm.w"])


def _cols(L, rank):
    """The 128 gate columns CTA ``rank`` owns, gate-major (r2d2_cluster.cuh: R2Clu::gcol)."""
    return np.concatenate([np.arange(k * L + 32 * rank, k * L + 32 * rank + 32) for k in range(4)])


def _keep(fx, L):
    return (~fx["inp"]["done"]).astype(np.float64).T.reshape(-1, 1)


def _bptt(buf, Wh, keep, B, S, L, drop=None, carry0=None):
    """dz of r2d2_lstm_bwd_cluster_kernel in float64, dh_in formed from its own dz_{t+1} as the kernel does; also the
    dc carry each sequence leaves after step 0.  ``drop`` = (t, owner, sender): the sender CTA's partial dh_in is
    missing at the owner's 32 units at step t; ``carry0``: the carry entering step S - 1 (a reset leaves zeros)."""
    dz = np.zeros((S * B, 4 * L))
    carry = np.zeros((B, L)) if carry0 is None else carry0
    for t in range(S - 1, -1, -1):
        r = slice(t * B, (t + 1) * B)
        si, tj, sf, so = (buf["gates"][r, k * L:(k + 1) * L] for k in range(4))
        tcv, cin, kt = buf["tc"][r], buf["cin"][r], keep[r]
        dh_next = dz[(t + 1) * B:(t + 2) * B] @ Wh.T if t < S - 1 else np.zeros((B, L))
        if drop is not None and t == drop[0]:
            own, snd = slice(32 * drop[1], 32 * drop[1] + 32), _cols(L, drop[2])
            dh_next[:, own] -= dz[(t + 1) * B:(t + 2) * B][:, snd] @ Wh[own][:, snd].T
        dh = buf["dhout"][r] + kt * dh_next
        dc = kt * carry + dh * so * (1 - tcv ** 2)
        dz[r] = np.concatenate([dc * tj * si * (1 - si), dc * si * (1 - tj ** 2), dc * cin * sf * (1 - sf),
                                dh * tcv * so * (1 - so)], 1)
        carry = dc * sf
    return dz, carry


def _mutate(fx, L, which):
    """(buffers, gradients) as the step would leave them with bug ``which``."""
    buf = {k: v.copy() for k, v in fx["buf"].items()}
    grads = {k: v.copy() for k, v in fx["grads"].items()}
    B, S = MUT_B[L], MUT_S
    W = _W(fx)
    Wx, Wh = W[:alp.XCAT], W[alp.XCAT:]
    bias = _np(fx["params"]["lstm.b"])
    if which == "late_store":               # rank 3 forms step t's gates from h_{t-2} (the state of step t - 1)
        cols = _cols(L, 3)
        z = buf["zx"][B:, cols] + bias[cols] + buf["hin"][:-B] @ Wh[:, cols]
        buf["gates"][B:, cols] = alp._gates(z, 32)
    elif which == "column_map_64":          # rank 5 reads its W_h columns through the 64-wide column map
        cols = _cols(L, 5)
        wrong = np.concatenate([np.arange(k * 64 + 32 * 5, k * 64 + 32 * 5 + 32) for k in range(4)])
        z = buf["zx"][:, cols] + bias[cols] + buf["hin"] @ Wh[:, wrong]
        buf["gates"][:, cols] = alp._gates(z, 32)
    elif which == "smem_segment":           # 512: rank 2 drops weights 56..127 (shared memory) of K segment 1
        cols, k = _cols(L, 2), slice(128 + 56, 256)
        z = buf["zx"][:, cols] + bias[cols] + buf["hin"] @ Wh[:, cols] - buf["hin"][:, k] @ Wh[k][:, cols]
        buf["gates"][:, cols] = alp._gates(z, 32)
    elif which == "bptt_missing_partial":   # sender 5's partial dh_in never reaches owner 2 at step 1
        buf["dz"] = _bptt(buf, Wh, _keep(fx, L), B, S, L, drop=(1, 2, 5))[0]
    elif which == "dc_carry_not_reset":     # one cluster walks both chunks and keeps the first chunk's carry
        _, left = _bptt(buf, Wh, _keep(fx, L), B, S, L)
        carry0 = np.zeros((B, L))
        carry0[MUT_R:] = left[:B - MUT_R]
        buf["dz"] = _bptt(buf, Wh, _keep(fx, L), B, S, L, carry0=carry0)[0]
    elif which == "hin_not_reset":          # step 0 of the second chunk reads the first chunk's last h
        buf["hin"][MUT_R:B] = buf["hin"][(S - 1) * B:(S - 1) * B + B - MUT_R]
    elif which == "zx_missing_partial":     # 512: split-K partial 1 of 8 is missing from N tile 5 of 8
        k, n = slice(424, 848), slice(5 * 256, 6 * 256)
        xcat = np.concatenate([buf["a3"], buf["emb"][fx["inp"]["pa"]]], axis=1)
        buf["zx"][:, n] -= xcat[:, k] @ Wx[k][:, n]
    elif which == "wgrad_h_rows_zero":      # the h rows [64, L) of lstm.w's gradient are never written
        grads["lstm.w"][alp.XCAT + 64:] = 0.0
    elif which == "q1_first_64_units":      # q1_fwd reads only the first 64 units of hout
        buf["q1"] = np.maximum(buf["hout"][:, :64] @ _np(fx["params"]["q1.w"])[:64] + _np(fx["params"]["q1.b"]), 0.0)
    return buf, grads


# (bug, width, kernel, tensor, what `where` must name)
MUTATIONS = [("late_store", 256, "r2d2_lstm_fwd", "gates", "rank3"),
             ("column_map_64", 256, "r2d2_lstm_fwd", "gates", "rank5"),
             ("smem_segment", 512, "r2d2_lstm_fwd", "gates", "rank2"),
             ("bptt_missing_partial", 256, "r2d2_lstm_bwd", "dz/o", ".rank2/"),
             ("dc_carry_not_reset", 256, "r2d2_lstm_bwd", "dz/ijf", ".rank"),
             ("hin_not_reset", 256, "r2d2_lstm_fwd", "hin[0]", ""),
             ("zx_missing_partial", 512, "lstm_x_fwd+reduce", "zx", ".n5/"),
             ("wgrad_h_rows_zero", 256, "lstm_wgrad", "lstm.w", "h."),
             ("q1_first_64_units", 256, "q1_fwd", "q1", "")]


@pytest.mark.parametrize("L", [256, 512])
def test_r2d2_wide_rows_pass_on_oracle_buffers(r2d2_wide, L):
    """Every row of check_r2d2 (and of check_r2d2_forward, the td_error check) passes on the oracle-consistent
    buffers, and the float64 BPTT the mutations re-run reproduces their dz: the mutations below start from a state
    every check accepts."""
    fx = r2d2_wide[L]
    rows = _rows(fx, L)
    assert len(rows) == len(alp.R2D2_KERNEL) + 4 + 3 + 6 + 2 + 1
    fwd, _ = alp.check_r2d2_forward({k: fx["buf"][k] for k in alp.R2D2_FWD_BUFFERS}, fx["params"], fx["batch"],
                                    MUT_B[L], MUT_S, MUT_A, L)
    assert len(fwd) == len(alp.R2D2_FWD_KERNEL) + 4 + 3
    bad = [(r["kernel"], r["tensor"], _excess(r)) for r in rows + fwd if not r["ok"]]
    assert not bad, bad
    dz, _ = _bptt(fx["buf"], _W(fx)[alp.XCAT:], _keep(fx, L), MUT_B[L], MUT_S, L)
    assert parity.rel_err(dz, fx["buf"]["dz"]) < TOL


@pytest.mark.parametrize("which,L,kernel,tensor,where", MUTATIONS)
def test_r2d2_wide_mutation_fails_its_row(r2d2_wide, which, L, kernel, tensor, where):
    fx = r2d2_wide[L]
    buf, grads = _mutate(fx, L, which)
    rows = {(r["kernel"], r["tensor"]): r for r in _rows(fx, L, buf, grads)}
    row = rows[(kernel, tensor)]
    assert _excess(row) >= 10, row
    assert where in row["where"], row
