"""Per-kernel float64 references of the Ape-X, A3C and R2D2 learner steps, fed from the step's own buffers.

The same check as tests/layer_parity.py (IMPALA), for the three learners that share the Adam handle: every reference is
computed from the device buffers its kernel read in the same step, with the oracle's layer functions
(``oracle.impala_torch``, which ``apex_torch`` / ``a3c_torch`` / ``r2d2_torch`` reuse) and torch autograd (a backward
kernel's upstream gradient is the GPU's own buffer, its ReLU masks the GPU's own activations).  The conv trunk and the
action embedding go through ``layer_parity.trunk_references``, shared with IMPALA.

Device conventions (csrc/apex.cu, csrc/r2d2.cu):
  * Ape-X / A3C: forward rows [0, B) are s with the previous action, rows [B, 2B) s' with the action; only the prefix
    Mb = B is backpropagated.  hid1 / hid2 / dhid2 / dhid1 stack the value (actor) half on top of the mean (critic)
    half; vstream is the value stream [M, A] (A3C: the logits), mstream the mean stream [M] (A3C: the value), policy
    the softmax of vstream; dq / dmean have 32 columns (A3C: dlogits / dv; dmean: column 0).
  * R2D2: rows are time-major, m = t*B + b, the batch is staged batch-major; all M = B*S rows receive gradient.  zx is
    the input half of the LSTM contraction ([a3 | emb] W[:3392], no bias); gates = [sigmoid(i) | tanh(j) |
    sigmoid(f + 1) | sigmoid(o)] of 64 columns each; hin / cin are the (masked) state each step read, tc = tanh(c_t),
    hout = h_t (un-masked).  The recurrence is checked one step at a time from the kernel's own stored state; its BPTT
    one step at a time from the GPU's own dz of the next step, with only the dc carry re-run (float64).

Bars (``apex_bars``, ``r2d2_bars``) come from the error model of each kernel's arithmetic (layer_parity's constants);
the loss kernels, whose outputs cancel (target - q, the advantage), are held per element to bounds derived from the
float32 rounding of the values they combine (``_td_bounds``, ``a3c_loss``).
"""
import numpy as np
import torch

import layer_parity as lp
from layer_parity import ELEM, FFMA_DOT, FLAT, TF32, TILE, VTRACE, _dense, _mask, _np, _t, time_major
from oracle import a3c_torch as at
from oracle import apex_torch as ax
from oracle import r2d2_torch as rt

U = 2.0 ** -24                  # float32 unit roundoff
R2L, R2G, R2H = 64, 256, 128    # R2D2 LSTM size, gate columns, q1 width
XCAT = FLAT + 256               # [a3 | emb] columns (both learners' first contraction)
TINY = 1e-300


def r2d2_bptt_bar(S):
    """dz of r2d2_lstm_bwd_kernel, per tensor and block: the K = 256 FFMA dot dz_{t+1} W_h^T (FFMA_DOT) plus the dc
    carry, which takes at most four float32 roundings per step (dh, dc, dc * sf and the gate product), each <= 2^-24 of
    the magnitudes involved, and is carried with the factor sf <= 1 over at most S steps."""
    return FFMA_DOT + 4 * S * U


# ------------------------------------------------------------------------------------------------------------------
# buffers
# ------------------------------------------------------------------------------------------------------------------
# name -> (rows, per-row shape) as in layer_parity.BUFFERS
APEX_BUFFERS = {
    "a1": ("M", (20, 20, 32)), "a2": ("M", (9, 9, 64)), "a3": ("M", (FLAT,)),
    "e1": ("A", (256,)), "emb": ("A", (256,)),
    "hid1": ("2M", (256,)), "hid2": ("2M", (256,)),
    "vstream": ("MA", ()), "mstream": ("M", ()), "policy": ("MA", ()),
    "dq": ("Mb", (32,)), "dmean": ("Mb", (32,)),
    "dhid2": ("2Mb", (256,)), "dhid1": ("2Mb", (256,)), "du": ("Mb", (256,)),
    "da3": ("Mb", (FLAT,)), "da2": ("Mb", (9, 9, 64)), "da1": ("Mb", (20, 20, 32)),
}
R2D2_BUFFERS = {
    "a1": ("M", (20, 20, 32)), "a2": ("M", (9, 9, 64)), "a3": ("M", (FLAT,)),
    "e1": ("A", (256,)), "emb": ("A", (256,)),
    "zx": ("M", (R2G,)), "gates": ("M", (R2G,)), "tc": ("M", (R2L,)), "hout": ("M", (R2L,)),
    "hin": ("M", (R2L,)), "cin": ("M", (R2L,)), "q1": ("M", (R2H,)), "q": ("MA", ()),
    "dq": ("M", (32,)), "dmean": ("M", (32,)), "dq1": ("M", (R2H,)), "dhout": ("M", (R2L,)), "dz": ("M", (R2G,)),
    "da3": ("M", (FLAT,)), "du": ("M", (256,)), "da2": ("M", (9, 9, 64)), "da1": ("M", (20, 20, 32)),
}


def read_buffers(eng, table, M, Mb, A):
    """Every buffer of ``table`` of the step the engine just ran, as float64 arrays in device layout."""
    out = {}
    for name, (rows, shp) in table.items():
        if rows == "MA":
            n, shape = M * A, (M, A)
        elif rows == "A":
            n, shape = A * int(np.prod(shp)), (A,) + shp
        else:
            r = {"M": M, "Mb": Mb, "2M": 2 * M, "2Mb": 2 * Mb}[rows]
            n, shape = r * int(np.prod(shp)), ((2, r // 2) if rows.startswith("2") else (r,)) + shp
        out[name] = eng.read_buffer(name, n).astype(np.float64).reshape(shape)
    return out


def _frames(u8):
    return (np.asarray(u8).astype(np.float32) / np.float32(255.0)).astype(np.float64)


def _P(p):
    return {k: v.detach().to(torch.float64) for k, v in p.items()}


# ------------------------------------------------------------------------------------------------------------------
# loss kernels
# ------------------------------------------------------------------------------------------------------------------
def _td_bounds(target, sav, diff, et, w, scale):
    """Per-element bounds of a float32 TD kernel: the target carries its own rounding ``et``, diff = target - sav one
    more rounding, the gradient g = -2 w diff * scale three more (|g| relative)."""
    ediff = et + U * (np.abs(target) + np.abs(sav))
    eg = 2 * w * scale * (ediff + 4 * U * np.abs(diff))
    return ediff, eg


def r2d2_td(mq, tq, batch, bi, gamma, B, S, A):
    """r2d2_td_kernel from the main / target q it read ([B, S, A], batch-major): the double-Q target with the argmax
    taken on ``mq`` itself (first maximum), value rescaling in float64, the window t in [bi, S - 1).  Returns the
    references and their per-element bounds (``bound/<name>``)."""
    Nt = S - bi - 1
    t = bi + np.arange(Nt)
    mq, tq = np.asarray(mq, np.float64), np.asarray(tq, np.float64)
    arg = np.argmax(mq[:, t + 1], axis=2)                                   # first maximum
    nsav = np.take_along_axis(tq[:, t + 1], arg[..., None], 2)[..., 0]
    act = np.asarray(batch["action"]).astype(np.int64)[:, t]
    sav = np.take_along_axis(mq[:, t], act[..., None], 2)[..., 0]
    disc = np.where(np.asarray(batch["done"]).astype(bool)[:, t], 0.0, gamma)
    r = np.asarray(batch["reward"], np.float32).astype(np.float64)[:, t]
    with torch.no_grad():
        target = _np(rt.vf_rescale(rt.vf_rescale_inv(_t(nsav)) * _t(disc) + _t(r)))
    diff = target - sav
    w = np.asarray(batch["weight"], np.float32).astype(np.float64)[:, None]
    scale = 1.0 / (Nt * B)
    g = -2.0 * w * diff * scale
    M = B * S
    dq, dmean = np.zeros((M, A)), np.zeros(M)
    eq, em = np.zeros((M, A)), np.zeros(M)
    ediff, eg = _td_bounds(target, sav, diff, U * np.abs(target), w, scale)
    rows = t[None, :] * B + np.arange(B)[:, None]
    dq[rows, act], dmean[rows] = g, -g
    eq[rows, act], em[rows] = eg, eg
    ref = dict(target_value=target, sav=sav, td=np.abs(diff.mean(axis=1)), loss=float(np.mean(w[:, 0] * (diff ** 2).mean(1))),
               dq=dq, dmean=dmean)
    # td: a float32 sum over the window (a lane loop and a warp tree: depth <= 8) of diffs that each carry ediff
    ref["bound/td"] = ediff.mean(1) + 8 * U * np.abs(diff).mean(1) + U * ref["td"]
    ref["bound/loss"] = float(np.mean(w[:, 0] * (2 * np.abs(diff) * ediff + 16 * U * diff ** 2).mean(1)))
    ref["bound/target_value"] = U * np.abs(target)
    ref["bound/sav"] = np.zeros_like(sav)                                   # a copy
    ref["bound/dq"], ref["bound/dmean"] = eq, em
    return ref


def apex_td(main_q, next_main_q, target_q, batch, gamma, clip, A):
    """apex_td_kernel from the q values it computed (``taps``): the argmax on ``next_main_q`` (first maximum), the
    target nsav * gamma (1 - done) + clip(r), the weighted loss and the head gradients."""
    mq, nq, tq = (np.asarray(x, np.float64) for x in (main_q, next_main_q, target_q))
    n = mq.shape[0]
    arg = np.argmax(nq, axis=1)
    nsav = tq[np.arange(n), arg]
    act = np.asarray(batch["action"]).astype(np.int64)
    sav = mq[np.arange(n), act]
    r = np.asarray(batch["reward"], np.float32).astype(np.float64)
    if clip:
        r = np.clip(r, -1.0, 1.0)
    disc = np.where(np.asarray(batch["done"]).astype(bool), 0.0, gamma)
    target = nsav * disc + r
    diff = target - sav
    w = np.asarray(batch["is_weight"], np.float32).astype(np.float64)
    g = -2.0 * w * diff / n
    dq = np.zeros((n, A))
    dq[np.arange(n), act] = g
    ediff, eg = _td_bounds(target, sav, diff, 2 * U * (np.abs(nsav * disc) + np.abs(r)), w, 1.0 / n)
    eq = np.zeros((n, A))
    eq[np.arange(n), act] = eg
    return dict(target_value=target, sav=sav, td=np.abs(diff), loss=float(np.mean(w * diff ** 2)), dq=dq, dmean=-g,
                **{"bound/target_value": 2 * U * (np.abs(nsav * disc) + np.abs(r)), "bound/sav": np.zeros(n),
                   "bound/td": ediff + U * np.abs(diff),
                   "bound/loss": float(np.mean(w * (2 * np.abs(diff) * ediff + 16 * U * diff ** 2))),
                   "bound/dq": eq, "bound/dmean": eg})


def a3c_loss(policy, value, next_value, batch, cfg):
    """a3c_loss_kernel from the policy and values it read: dlogits / dv by autograd of the oracle's a2c loss through a
    softmax of log(policy) (softmax(log p) = p, so the gradient is the kernel's p (dp - sum p dp)), the advantage and
    the three loss terms.  ``cfg``: discount_factor, baseline_loss_coef, entropy_coef, reward_clipping (the values the
    kernel was given)."""
    p = np.asarray(policy, np.float64)
    n, A = p.shape
    r = np.asarray(batch["reward"], np.float32).astype(np.float64)
    if cfg["reward_clipping"] == "abs_one":
        cr, ecr = np.clip(r, -1.0, 1.0), np.zeros(n)
    else:
        sq = np.tanh(r / 5.0)
        cr = np.where(r < 0, 0.3 * sq, sq) * 5.0
        ecr = 8 * U * np.abs(cr)            # tanhf (<= 2 ulp), the divide and two products
    done = torch.from_numpy(np.asarray(batch["done"]).astype(bool))
    disc = (~done).to(torch.float64) * cfg["discount_factor"]
    lg = _t(np.log(p), True)
    v = _t(value, True)
    nv = _t(next_value)
    pol = torch.softmax(lg, dim=1)
    a = torch.from_numpy(np.asarray(batch["action"]).astype(np.int64))
    pi = at.compute_policy_loss(pol, a, v, nv, disc, _t(cr), A)         # (for the gradients)
    bl = at.compute_baseline_loss(v, nv, disc, _t(cr))
    en = at.compute_entropy_loss(pol)
    total = pi + bl * cfg["baseline_loss_coef"] + en * cfg["entropy_coef"]
    dlg, dv = torch.autograd.grad(total, (lg, v))
    adv = cr + _np(disc) * np.asarray(next_value, np.float64) - np.asarray(value, np.float64)
    # the advantage: three float32 roundings of the magnitudes it combines
    eadv = ecr + 4 * U * (np.abs(cr) + np.abs(np.asarray(next_value)) + np.abs(np.asarray(value)))
    dlg = _np(dlg)
    bc = cfg["baseline_loss_coef"]
    pa = p[np.arange(n), np.asarray(batch["action"]).astype(np.int64)]
    plogp = np.where(p > 0, p * np.log(np.where(p > 0, p, 1.0)), 0.0)
    # the loss terms of the stored policy itself (the kernel does not renormalise it: at min p ~ 1e-20 a float32
    # policy sums to 1 only within ~A ulps, which moves p log p of the largest p by as much as its own size)
    return dict(adv=adv, dq=dlg, dmean=_np(dv), pi_loss=float(-np.mean(adv * pa)), baseline_loss=float(_np(bl)),
                entropy=float(np.mean(plogp.sum(1))),
                **{"bound/adv": eadv,
                   # a softmax backward of <= 32 terms with a log each (the V-trace kernel's bar), plus the advantage's
                   # error, which reaches dlogit_k with the weight p_k (1 - p_k) / n <= 1 / n
                   "bound/dq": np.broadcast_to(VTRACE * np.max(np.abs(dlg)) + eadv[:, None] / n, dlg.shape),
                   "bound/dmean": 2 * bc / n * (eadv + 4 * U * np.abs(adv)),
                   # float32 sums of n (and n * A) terms: depth <= 64 with the warp trees and the lane loops
                   "bound/pi_loss": float(np.mean(eadv * pa + 64 * U * np.abs(adv * pa))),
                   "bound/baseline_loss": float(np.mean(2 * np.abs(adv) * eadv + 64 * U * adv ** 2)),
                   "bound/entropy": float(np.mean(96 * U * np.abs(plogp).sum(1)))})


# ------------------------------------------------------------------------------------------------------------------
# Ape-X / A3C
# ------------------------------------------------------------------------------------------------------------------
def stream_names(algo):
    return ("value", "mean") if algo == "apex" else ("actor", "critic")


def apex_inputs(batch):
    """The staged batch in device row order: [s ; s'] / 255 and [previous action ; action]."""
    x = _frames(np.concatenate([batch["state"], batch["next_state"]]))
    pa = np.concatenate([batch["previous_action"], batch["action"]]).astype(np.int64)
    return dict(x=x, pa=pa)


def apex_references(buf, p, batch, B, A, algo):
    """{output: float64 reference} of the Ape-X (``algo`` = "apex") or A3C ("a3c") network forward and head / trunk
    backward, each from the GPU buffers its kernel read.  The loss kernels are ``apex_td`` / ``a3c_loss``."""
    inp = apex_inputs(batch)
    P = _P(p)
    W = {k: _np(v) for k, v in P.items()}
    ref = lp.trunk_references(buf, P, inp["x"], inp["pa"], A, B)
    sv, sm = stream_names(algo)
    cat = np.concatenate([buf["a3"], buf["emb"][inp["pa"]]], axis=1)
    with torch.no_grad():
        ref["hid1"] = np.stack([_np(torch.relu(_t(cat) @ P[s + "1.w"] + P[s + "1.b"])) for s in (sv, sm)])
        ref["hid2"] = np.stack([_np(torch.relu(_t(buf["hid1"][z]) @ P[s + "2.w"] + P[s + "2.b"]))
                                for z, s in enumerate((sv, sm))])
        ref["vstream"] = _np(_t(buf["hid2"][0]) @ P[sv + "3.w"] + P[sv + "3.b"])
        ref["mstream"] = _np(_t(buf["hid2"][1]) @ P[sm + "3.w"] + P[sm + "3.b"])[:, 0]
        ref["policy"] = _np(torch.softmax(_t(buf["vstream"]), dim=1))      # same kernel: softmax of what it stored
    # ---- heads backward over the first B rows ---------------------------------------------------------------------
    h1, h2 = buf["hid1"][:, :B], buf["hid2"][:, :B]
    dxv, ref[sv + "3.w"], ref[sv + "3.b"] = _dense(h2[0], W[sv + "3.w"], W[sv + "3.b"], buf["dq"][:, :A])
    dxm, ref[sm + "3.w"], ref[sm + "3.b"] = _dense(h2[1], W[sm + "3.w"], W[sm + "3.b"], buf["dmean"][:, :1])
    ref["dhid2"] = np.stack([dxv, dxm]) * _mask(h2)
    dh1, dcat = [], 0.0
    for z, s in enumerate((sv, sm)):
        dx, ref[s + "2.w"], ref[s + "2.b"] = _dense(h1[z], W[s + "2.w"], W[s + "2.b"], buf["dhid2"][z])
        dh1.append(dx * _mask(h1[z]))
        dx, ref[s + "1.w"], ref[s + "1.b"] = _dense(cat[:B], W[s + "1.w"], W[s + "1.b"], buf["dhid1"][z])
        dcat = dcat + dx
    ref["dhid1"] = np.stack(dh1)
    ref["da3"] = dcat[:, :FLAT] * _mask(buf["a3"][:B])
    ref["du"] = dcat[:, FLAT:]
    return ref


# ------------------------------------------------------------------------------------------------------------------
# R2D2
# ------------------------------------------------------------------------------------------------------------------
def r2d2_inputs(batch):
    """The staged batch in device row order (time-major): frames / 255, previous action; h0 / c0 per sequence, done."""
    return dict(x=_frames(time_major(batch["state"])), pa=time_major(batch["previous_action"]).astype(np.int64),
                h0=np.asarray(batch["h"], np.float32)[:, 0].astype(np.float64),
                c0=np.asarray(batch["c"], np.float32)[:, 0].astype(np.float64),
                done=np.asarray(batch["done"]).astype(bool))


def _gates(z):
    i, j, f, o = (z[:, k * R2L:(k + 1) * R2L] for k in range(4))
    return np.concatenate([1 / (1 + np.exp(-i)), np.tanh(j), 1 / (1 + np.exp(-(f + 1.0))), 1 / (1 + np.exp(-o))], 1)


def r2d2_references(buf, p, batch, B, S, A):
    """{output: float64 reference} of the R2D2 main-scope forward (trunk, lstm_x_fwd, the recurrence step by step from
    the kernel's stored state, q1, q) and the whole backward, each from the GPU buffers its kernel read.  The TD kernel
    is ``r2d2_td``.  Adds ``z`` (the recurrence's pre-activation, for bounds and regime checks) and ``cnext``: the
    reference c_t * (1 - done_t) of every row but the last step, which the next step's ``cin`` must hold."""
    inp = r2d2_inputs(batch)
    M = B * S
    P = _P(p)
    W = {k: _np(v) for k, v in P.items()}
    ref = lp.trunk_references(buf, P, inp["x"], inp["pa"], A, M)
    xcat = np.concatenate([buf["a3"], buf["emb"][inp["pa"]]], axis=1)
    Wx, Wh = W["lstm.w"][:XCAT], W["lstm.w"][XCAT:]
    ref["zx"] = xcat @ Wx
    # ---- recurrence, one step at a time from the stored state ----------------------------------------------------------
    z = buf["zx"] + W["lstm.b"] + buf["hin"] @ Wh
    g = _gates(z)
    si, tj, sf, so = (g[:, k * R2L:(k + 1) * R2L] for k in range(4))
    c = sf * buf["cin"] + si * tj
    ref["z"], ref["gates"], ref["c"] = z, g, c
    ref["tc"] = np.tanh(c)
    ref["hout"] = so * ref["tc"]
    keep = (~inp["done"]).astype(np.float64).T.reshape(M, 1)           # time-major rows
    ref["cnext"] = (c * keep)[:M - B]
    # ---- head ------------------------------------------------------------------------------------------------------
    ref["q1"] = np.maximum(buf["hout"] @ W["q1.w"] + W["q1.b"], 0.0)
    ref["q"] = (buf["q1"] @ W["value.w"] + W["value.b"]) - (buf["q1"] @ W["mean.w"] + W["mean.b"])
    # ---- backward ---------------------------------------------------------------------------------------------------
    dxv, ref["value.w"], ref["value.b"] = _dense(buf["q1"], W["value.w"], W["value.b"], buf["dq"][:, :A])
    dxm, ref["mean.w"], ref["mean.b"] = _dense(buf["q1"], W["mean.w"], W["mean.b"], buf["dmean"][:, :1])
    ref["dq1"] = (dxv + dxm) * _mask(buf["q1"])
    ref["dhout"], ref["q1.w"], ref["q1.b"] = _dense(buf["hout"], W["q1.w"], W["q1.b"], buf["dq1"])
    # BPTT: dz_t from the GPU's dhout_t, its forward buffers and its own dz_{t+1}; only the dc carry is re-run
    gg = buf["gates"]
    gi, gj, gf, go = (gg[:, k * R2L:(k + 1) * R2L] for k in range(4))
    dz = np.zeros((M, R2G))
    carry = np.zeros((B, R2L))
    for t in range(S - 1, -1, -1):
        r = slice(t * B, (t + 1) * B)
        kt = keep[r]
        dh = buf["dhout"][r] + (kt * (buf["dz"][(t + 1) * B:(t + 2) * B] @ Wh.T) if t < S - 1 else 0.0)
        dc = kt * carry + dh * go[r] * (1 - buf["tc"][r] ** 2)
        dz[r] = np.concatenate([dc * gj[r] * gi[r] * (1 - gi[r]), dc * gi[r] * (1 - gj[r] ** 2),
                                dc * buf["cin"][r] * gf[r] * (1 - gf[r]), dh * buf["tc"][r] * go[r] * (1 - go[r])], 1)
        carry = dc * gf[r]
    ref["dz"] = dz
    dx, ref["lstm.w"], ref["lstm.b"] = _dense(np.concatenate([xcat, buf["hin"]], 1), W["lstm.w"], W["lstm.b"], buf["dz"])
    ref["da3"] = dx[:, :FLAT] * _mask(buf["a3"])
    ref["du"] = dx[:, FLAT:XCAT]
    return ref


def r2d2_recurrence_bounds(ref, cin):
    """Per-element bounds of gates / tc / hout / cnext: ``layer_parity.lstm_bounds`` with the K = 64 FFMA dot product
    h_in W_h (and the add of zx and the bias) as the pre-activation bar; tc = tanh(c) carries c's bound with its
    derivative."""
    b = lp.lstm_bounds(dict(z=ref["z"], gates=ref["gates"], c1=ref["c"]), cin, FFMA_DOT)
    tc = ref["tc"]
    etc = (1 - tc ** 2) * b["c1"] + b["c1"] ** 2 + ELEM
    return {"gates": b["gates"], "tc": etc, "hout": b["h1"], "cnext": b["c1"][:ref["cnext"].shape[0]]}


# ------------------------------------------------------------------------------------------------------------------
# metric
# ------------------------------------------------------------------------------------------------------------------
def r2d2_blocks(name, ref):
    """Natural sub-tensors of an R2D2 output: the i/j/f/o column blocks (64 wide) of zx / gates / dz / lstm.w, the a3 /
    emb / h row segments of lstm.w; every other output as in ``layer_parity.blocks``."""
    if name in ("zx", "gates", "dz"):
        return [("%s/r%d" % (g, s.start), (s, slice(k * R2L, (k + 1) * R2L)))
                for k, g in enumerate("ijfo") for s in lp._row_tiles(ref.shape[0])]
    if name == "lstm.w":
        segs = (("a3", 0, FLAT), ("emb", FLAT, XCAT), ("h", XCAT, XCAT + R2L))
        return [("%s.%s/r%d" % (sg, g, r0), (slice(r0, min(r0 + TILE, hi)), slice(k * R2L, (k + 1) * R2L)))
                for sg, lo, hi in segs for r0 in range(lo, hi, TILE) for k, g in enumerate("ijfo")]
    if name == "lstm.b":
        return [(g, (slice(k * R2L, (k + 1) * R2L),)) for k, g in enumerate("ijfo")]
    return lp.blocks(name, ref)


def bound_row(kernel, name, got, ref, bound):
    """A row held per element to ``bound`` (the ratio is reported; the per-tensor / block errors for information)."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    d = np.abs(got - ref)
    ratio = float(np.max(d / np.maximum(bound, TINY))) if d.size else 0.0
    if not np.all(np.isfinite(got)):
        ratio = float("inf")
    mx = float(np.max(np.abs(ref))) if ref.size else 0.0
    e = float(np.max(d)) / max(mx, 1e-30) if d.size else 0.0
    return dict(kernel=kernel, tensor=name, err=e, block=e, where="", bar="per-element bound", bound_ratio=ratio,
                ok=bool(ratio <= 1.0))


def bar_row(kernel, name, got, ref, bar, blocks_of=None):
    e, blk, where = lp.errors(name, got, ref, blocks_of)
    return dict(kernel=kernel, tensor=name, err=e, block=blk, where=where, bar=bar, ok=bool(e <= bar and blk <= bar))


def exact_row(kernel, name, got, ref):
    """A bitwise check (float32 values compared as float64)."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    bad = int(np.sum(got != ref))
    return dict(kernel=kernel, tensor=name, err=float(bad), block=float(bad), where="%d elements differ" % bad,
                bar="exact", ok=bad == 0)


TRUNK_KERNEL = {"a1": "conv1_fwd", "a2": "conv2_fwd", "a3": "conv3_fwd", "e1": "emb_fwd", "emb": "emb_fwd",
                "da2": "conv3_dgrad", "da1": "conv2_dgrad", "emb1.w": "emb_bwd", "emb1.b": "emb_bwd",
                "emb2.w": "emb_bwd", "emb2.b": "emb_bwd", "conv3.w": "conv3_wgrad+reduce",
                "conv3.b": "conv3_wgrad+reduce", "conv2.w": "conv2_wgrad+reduce", "conv2.b": "conv2_wgrad+reduce",
                "conv1.w": "conv1_wgrad+reduce", "conv1.b": "conv1_wgrad+reduce"}
# trunk bars in math modes 1 and 2 (3xTF32 or FFMA GEMMs; layer_parity.bars), the embedding as for IMPALA
TRUNK_BAR = {k: TF32 for k in TRUNK_KERNEL}
TRUNK_BAR.update(e1=ELEM, emb=FFMA_DOT)


def apex_kernels(algo):
    sv, sm = stream_names(algo)
    k = dict(TRUNK_KERNEL)
    k.update({"hid1": "heads_l1_fwd+apex_hid1", "hid2": "heads_l2_fwd", "vstream": "heads_out_fwd",
              "mstream": "heads_out_fwd", "policy": "heads_out_fwd", "dhid2": "heads_out_bwd",
              "dhid1": "heads_l2_dgrad", "da3": "heads_l1_dgrad", "du": "heads_l1_dgrad",
              sv + "3.w": "value3_wgrad", sv + "3.b": "value3_wgrad", sm + "3.w": "mean3_wgrad",
              sm + "3.b": "mean3_wgrad"})
    for s in (sv, sm):
        k.update({s + "2.w": "heads_l2_wgrad", s + "2.b": "heads_l2_wgrad", s + "1.w": "heads_l1_wgrad",
                  s + "1.b": "heads_l1_wgrad"})
    return k


def apex_bars(algo):
    b = {k: TF32 for k in apex_kernels(algo)}
    b.update(TRUNK_BAR)
    b.update(vstream=FFMA_DOT, mstream=FFMA_DOT, policy=ELEM, dhid2=FFMA_DOT)
    return b


R2D2_KERNEL = dict(TRUNK_KERNEL)
R2D2_KERNEL.update({"zx": "lstm_x_fwd+reduce", "q1": "q1_fwd", "q": "r2d2_out", "dq1": "r2d2_out_bwd",
                    "dhout": "q1_dgrad", "dz": "r2d2_lstm_bwd", "da3": "lstm_dgrad", "du": "lstm_dgrad",
                    "value.w": "value_wgrad", "value.b": "value_wgrad", "mean.w": "mean_wgrad",
                    "mean.b": "mean_wgrad", "q1.w": "q1_wgrad", "q1.b": "q1_wgrad", "lstm.w": "lstm_wgrad",
                    "lstm.b": "lstm_wgrad(bias reduce)"})


def r2d2_bars(S):
    b = {k: TF32 for k in R2D2_KERNEL}
    b.update(TRUNK_BAR)
    b.update(q=FFMA_DOT, dq1=FFMA_DOT, dz=r2d2_bptt_bar(S))
    return b


# ------------------------------------------------------------------------------------------------------------------
# comparison of one step
# ------------------------------------------------------------------------------------------------------------------
def check_apex(buf, grads, p, batch, taps, out, B, A, algo, cfg):
    """Rows (dict(kernel, tensor, err, block, where, bar, ok)) of every checked output of one Ape-X / A3C step.
    ``taps`` / ``out``: what the handle reported (q taps / losses); ``cfg``: the learner's loss settings."""
    ref = apex_references(buf, p, batch, B, A, algo)
    kern, bar = apex_kernels(algo), apex_bars(algo)
    got = dict(buf)
    got.update(grads)
    rows = [bar_row(kern[k], k, got[k], ref[k], bar[k]) for k in kern]
    gamma = float(np.float32(cfg["discount_factor"]))
    if algo == "apex":
        v, m = buf["vstream"], buf["mstream"]
        for name, sl in (("main_q", slice(0, B)), ("next_main_q", slice(B, 2 * B))):
            q = v[sl] - m[sl, None]
            rows.append(bound_row("apex_td", name, taps[name], q, U * np.abs(q)))
        td = apex_td(taps["main_q"], taps["next_main_q"], taps["target_q"], batch, gamma,
                     cfg["reward_clipping"] == "abs_one", A)
        gtd = dict(target_value=taps["target_value"], sav=taps["state_action_value"], td=out["td"], loss=out["loss"],
                   dq=buf["dq"][:, :A], dmean=buf["dmean"][:, 0])
        for k in ("target_value", "sav", "td", "loss", "dq", "dmean"):
            rows.append(bound_row("apex_td", k, gtd[k], td[k], td["bound/" + k]))
    else:
        ls = a3c_loss(buf["policy"][:B], buf["mstream"][:B], buf["mstream"][B:], batch,
                      dict(cfg, discount_factor=gamma))
        gl = dict(adv=taps["advantage"], dq=buf["dq"][:, :A], dmean=buf["dmean"][:, 0], pi_loss=out["pi_loss"],
                  baseline_loss=out["baseline_loss"], entropy=out["entropy"])
        for k in ("adv", "dq", "dmean", "pi_loss", "baseline_loss", "entropy"):
            rows.append(bound_row("a3c_loss", {"dq": "dlogits", "dmean": "dv"}.get(k, k), gl[k], ls[k], ls["bound/" + k]))
    return rows, ref


def check_r2d2(buf, grads, p, batch, taps, out, B, S, bi, A, gamma):
    """Rows of every checked output of one R2D2 step (see check_apex), the exact checks of the recurrence's state
    hand-over and of the gradient rows outside the loss window included."""
    M = B * S
    ref = r2d2_references(buf, p, batch, B, S, A)
    inp = r2d2_inputs(batch)
    got = dict(buf)
    got.update(grads)
    got["cnext"] = buf["cin"][B:]
    bar = r2d2_bars(S)
    rows = [bar_row(R2D2_KERNEL[k], k, got[k], ref[k], bar[k], r2d2_blocks) for k in R2D2_KERNEL]
    eb = r2d2_recurrence_bounds(ref, buf["cin"])
    for k in ("gates", "tc", "hout", "cnext"):
        rows.append(bound_row("r2d2_lstm_fwd", k, got[k], ref[k], eb[k]))
    keep = (~inp["done"]).astype(np.float64).T.reshape(M, 1)
    rows.append(exact_row("r2d2_lstm_fwd", "hin[0]", buf["hin"][:B], inp["h0"]))
    rows.append(exact_row("r2d2_lstm_fwd", "cin[0]", buf["cin"][:B], inp["c0"]))
    rows.append(exact_row("r2d2_lstm_fwd", "hin[t+1]", buf["hin"][B:], (buf["hout"] * keep)[:M - B]))
    td = r2d2_td(taps["main_q"], taps["target_q"], batch, bi, gamma, B, S, A)
    gtd = dict(target_value=taps["target_value"], sav=taps["state_action_value"], td=out["td"], loss=out["loss"],
               dq=buf["dq"][:, :A], dmean=buf["dmean"][:, 0])
    for k in ("target_value", "sav", "td", "loss", "dq", "dmean"):
        rows.append(bound_row("r2d2_td", k, gtd[k], td[k], td["bound/" + k]))
    # rows outside the loss window and every column >= A (dmean: >= 1) carry exactly zero
    t = np.arange(M) // B
    outside = (t < bi) | (t >= S - 1)
    rows.append(exact_row("r2d2_td", "dq/outside", np.concatenate([buf["dq"][outside].ravel(), buf["dq"][:, A:].ravel()]),
                          0.0))
    rows.append(exact_row("r2d2_td", "dmean/outside",
                          np.concatenate([buf["dmean"][outside].ravel(), buf["dmean"][:, 1:].ravel()]), 0.0))
    return rows, ref


# ------------------------------------------------------------------------------------------------------------------
# one step on the GPU
# ------------------------------------------------------------------------------------------------------------------
TRAIN_STEPS, TRAIN_LR = 20, 1e-3        # Adam at 10x the default rate: every parameter moves by up to ~2e-2
SCALE_LSTM = 60.0                       # R2D2 saturated: |z| > 4 for about 40 % of the gates (x20: 2.5 %)
BIG_RETURN = 300.0                      # rewards and target q in the hundreds (h and h^-1 at large |x|)
PEAK_LOGIT = 45.0                       # A3C peaked: logits spread over 45, min p ~ e^-45 ~ 3e-20
APEX_REGIMES = ("init", "trained", "large_returns", "ties")
A3C_REGIMES = ("init", "trained", "peaked")
R2D2_REGIMES = ("init", "trained", "saturated", "done_heavy", "large_returns", "ties")


def _train(eng, stage, steps):
    for s in range(steps):
        stage(10_000 + s)
        eng.step(0)


def _moved(flat0, flat, unflatten):
    flat = flat.astype(np.float64)
    p = unflatten(flat)
    return dict(param_moved_rel_l2=float(np.linalg.norm(flat - flat0) / np.linalg.norm(flat0)),
                biases_nonzero=all(bool(p[k].abs().max() > 0) for k in p if k.endswith(".b")))


def run_apex_case(algo, mode, B, A, regime, seed=4242):
    """One step of a fresh Ape-X (``algo`` = "apex") or A3C learner in ``regime``; returns (rows, facts) as
    layer_parity.run_case."""
    from distributed_reinforcement_learning_b200.a3c_learner import NativeA3CLearner
    from distributed_reinforcement_learning_b200.apex_learner import MAIN, TARGET, NativeApexLearner
    mod = ax if algo == "apex" else at
    kw = dict(num_action=A)
    params = mod.init_params(0, torch.float32, **kw)
    lr = TRAIN_LR if regime == "trained" else mod.DEFAULT_CFG["start_learning_rate"]
    clip = "none" if regime == "large_returns" else "abs_one"
    sv, sm = stream_names(algo)
    if regime == "ties":            # two identical value3 columns, raised above the others: exact ties at the maximum
        params[sv + "3.w"][:, 1] = params[sv + "3.w"][:, 0]
        params[sv + "3.b"][:2] = 1.0
    if regime == "peaked":
        params[sv + "3.b"] = torch.linspace(0.0, -PEAK_LOGIT, A, dtype=torch.float32)
    facts = {}
    if algo == "apex":
        target = ax.init_params(1, torch.float32, **kw)
        if regime == "large_returns":
            target["value3.b"] = torch.full((A,), BIG_RETURN, dtype=torch.float32)
        eng = NativeApexLearner(batch=B, num_action=A, math_mode=mode, reward_clipping=clip, start_learning_rate=lr)
        cfg = dict(discount_factor=ax.DEFAULT_CFG["discount_factor"], reward_clipping=clip)
    else:
        eng = NativeA3CLearner(batch=B, num_action=A, math_mode=mode, start_learning_rate=lr)
        cfg = {k: at.DEFAULT_CFG[k] for k in ("discount_factor", "baseline_loss_coef", "entropy_coef",
                                              "reward_clipping")}

    def batch_of(s):
        b = ax.make_transitions(B, A=A, seed=s)
        if regime == "large_returns":
            b["reward"] = (b["reward"] * BIG_RETURN).astype(np.float32)
        return b

    def stage(s):
        b = batch_of(s)
        eng.stage(0, *[b[k] for k in (ax.TRAIN_FIELDS if algo == "apex" else at.TRAIN_FIELDS)])
        return b
    try:
        flat0 = mod.flatten_params(params)
        if algo == "apex":
            eng.set_params(flat0, MAIN)
            eng.set_params(ax.flatten_params(target), TARGET)
        else:
            eng.set_params(flat0)
        if regime == "trained":
            _train(eng, stage, TRAIN_STEPS)
            facts.update(_moved(flat0.astype(np.float64), eng.get_params(),
                                lambda f: mod.unflatten_params(f, torch.float64, **kw)))
        p = mod.unflatten_params(eng.get_params(), torch.float64, **kw)
        batch = stage(seed)
        if algo == "apex":
            o, td = eng.step(0)
            out = dict(o, td=td)
        else:
            out = eng.step(0)
        taps = eng.taps()
        buf = read_buffers(eng, APEX_BUFFERS, 2 * B, B, A)
        grads = {k: v.numpy() for k, v in mod.unflatten_params(eng.get_grads(), torch.float64, **kw).items()}
    finally:
        eng.close()
    rows, ref = check_apex(buf, grads, p, batch, taps, out, B, A, algo, cfg)
    facts["finite"] = bool(all(np.all(np.isfinite(v)) for v in list(buf.values()) + list(grads.values())))
    if algo == "apex":
        nq = taps["next_main_q"]
        facts["tie_rows"] = int(np.sum(nq.max(1) == np.sort(nq, 1)[:, -2]))
        facts["target_abs_max"] = float(np.abs(taps["target_value"]).max())
    else:
        facts["policy_min"] = float(buf["policy"].min())
    return rows, facts


def run_r2d2_case(mode, B, S, bi, A, C, regime, seed=2468):
    """One step of a fresh R2D2 learner in ``regime``; returns (rows, facts) as layer_parity.run_case."""
    import r2d2_parity
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET, NativeR2D2Learner
    kw = dict(num_action=A, lstm_size=R2L, input_shape=(84, 84, C))
    params = rt.init_params(0, torch.float32, **kw)
    target = rt.init_params(1, torch.float32, **kw)
    if regime == "saturated":
        params["lstm.w"] = params["lstm.w"] * SCALE_LSTM
    if regime == "large_returns":
        target["value.b"] = torch.full((A,), BIG_RETURN, dtype=torch.float32)
    if regime == "ties":            # two identical value columns, raised above the others: exact ties at the maximum
        params["value.w"][:, 1] = params["value.w"][:, 0]
        params["value.b"][:2] = 1.0
    done_rate, done_ends = (0.3, True) if regime == "done_heavy" else (None, False)
    lr = TRAIN_LR if regime == "trained" else rt.LR
    eng = NativeR2D2Learner(batch=B, seq_len=S, burn_in=bi, num_action=A, input_shape=(84, 84, C), math_mode=mode,
                            learning_rate=lr)

    def stage(s):
        b = r2d2_parity.make_batch(B, S, A, C, s, done_rate, done_ends)
        if regime == "large_returns":
            b["reward"] = (b["reward"] * BIG_RETURN).astype(np.float32)
        eng.stage(0, b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"], b["done"],
                  b["weight"])
        return b
    facts = {}
    try:
        flat0 = rt.flatten_params(params)
        eng.set_params(flat0, MAIN)
        eng.set_params(rt.flatten_params(target), TARGET)
        if regime == "trained":
            _train(eng, stage, TRAIN_STEPS)
            facts.update(_moved(flat0.astype(np.float64), eng.get_params(),
                                lambda f: rt.unflatten_params(f, torch.float64, **kw)))
        p = rt.unflatten_params(eng.get_params(), torch.float64, **kw)
        batch = stage(seed)
        o, td = eng.step(0)
        taps = eng.taps()
        buf = read_buffers(eng, R2D2_BUFFERS, B * S, B * S, A)
        grads = {k: v.numpy() for k, v in rt.unflatten_params(eng.get_grads(), torch.float64, **kw).items()}
    finally:
        eng.close()
    rows, ref = check_r2d2(buf, grads, p, batch, taps, dict(o, td=td), B, S, bi, A,
                           float(np.float32(rt.DEFAULT_CFG["discount_factor"])))
    facts["finite"] = bool(all(np.all(np.isfinite(v)) for v in list(buf.values()) + list(grads.values())))
    facts["z_abs_gt4"] = float(np.mean(np.abs(ref["z"]) > 4))
    facts["c_abs_max"] = float(np.abs(ref["c"]).max())
    facts["done_rate"] = float(np.mean(batch["done"]))
    facts["done_ends"] = bool(batch["done"][:, 0].all() and batch["done"][:, -1].all())
    facts["target_abs_max"] = float(np.abs(taps["target_q"]).max())        # what h^-1 reads
    mq = taps["main_q"][:, bi + 1:]
    facts["tie_rows"] = int(np.sum(mq.max(2) == np.sort(mq, 2)[..., -2]))
    return rows, facts


def launch_facts():
    """The split-K counts the library plans (drl_debug_apex_launch_plan / drl_debug_r2d2_launch_plan) for a shape:
    ``apex(B, mode)`` -> dict(heads_l1_fwd, conv1_wgrad, conv2_wgrad, conv3_wgrad); ``r2d2(B, S, C, mode)`` -> the same
    with lstm_x_fwd for heads_l1_fwd."""
    import ctypes
    from distributed_reinforcement_learning_b200 import _native as N

    def apex(B, mode):
        out = (ctypes.c_int32 * 4)()
        N.check(N.lib.drl_debug_apex_launch_plan(B, mode, out))
        return dict(heads_l1_fwd=out[0], conv1_wgrad=out[1], conv2_wgrad=out[2], conv3_wgrad=out[3])

    def r2d2(B, S, C, mode):
        out = (ctypes.c_int32 * 4)()
        N.check(N.lib.drl_debug_r2d2_launch_plan(B, S, C, mode, out))
        return dict(lstm_x_fwd=out[0], conv1_wgrad=out[1], conv2_wgrad=out[2], conv3_wgrad=out[3])
    return apex, r2d2
