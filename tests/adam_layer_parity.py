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
    sigmoid(f + 1) | sigmoid(o)] of L columns each (lstm_size L = 64, 256 or 512); hin / cin are the (masked) state each
    step read, tc = tanh(c_t), hout = h_t (un-masked).  The recurrence is checked one step at a time from the kernel's
    own stored state; its BPTT one step at a time from the GPU's own dz of the next step, with only the dc carry re-run
    (float64).  At L = 256 / 512 the recurrence runs on a thread-block cluster (csrc/r2d2_cluster.cuh): CTA rank r owns
    units [32 r, 32 r + 32) of every gate, and failures are labelled by that rank and by the 256-wide N tile of the LSTM
    GEMMs.

Bars (``apex_bars``, ``r2d2_bars``) come from the error model of each kernel's arithmetic (layer_parity's constants);
the loss kernels, whose outputs cancel (target - q, the advantage), are held per element to bounds derived from the
float32 rounding of the values they combine (``_td_bounds``, ``a3c_loss``).
"""
import functools
import math

import numpy as np
import torch

import layer_parity as lp
from layer_parity import ELEM, FFMA_DOT, FLAT, TF32, TILE, VTRACE, _dense, _mask, _np, _t, time_major
from oracle import a3c_torch as at
from oracle import apex_torch as ax
from oracle import r2d2_torch as rt

U = 2.0 ** -24                  # float32 unit roundoff
R2L, R2G, R2H = 64, 256, 128    # R2D2 LSTM size (the default), its gate columns, q1 width
R2_SIZES = (64, 256, 512)       # the widths the R2D2 learner supports
R2_NTILE = 256                  # N tile of the LSTM GEMMs (lstm_x_fwd, lstm_wgrad)
XCAT = FLAT + 256               # [a3 | emb] columns (both learners' first contraction)
TINY = 1e-300


def gamma(n):
    """gamma_n = n u / (1 - n u): the relative bound of a float32 sum of products that passes through n roundings."""
    return n * U / (1 - n * U)


def r2d2_fwd_terms(L):
    """Roundings a term of the cluster forward's pre-activation passes through (r2d2_lstm_fwd_cluster_kernel): a chain
    of 128 FFMAs per K segment, the KS - 1 adds of the KS = L / 128 segment sums, and the add of bias + zx."""
    return 128 + L // 128 + 1


def r2d2_bwd_terms(L):
    """Roundings a term of dh = dhout + dz_{t+1} W_h^T passes through in r2d2_lstm_bwd_cluster_kernel: each CTA's chain
    of 128 FFMAs over its gate columns, the CL = L / 32 partials added by the owner in rank order, and the add of
    dhout."""
    return 128 + L // 32 + 1


def r2d2_bptt_bar(S, L=R2L):
    """dz of the R2D2 BPTT kernel, per tensor and block (at L > 64 the i / j / f blocks; the o block is held per
    element, see r2d2_recurrence_bounds): the dot product dh = dhout + dz_{t+1} W_h^T plus the dc carry, which takes at
    most four float32 roundings per step (dh, dc, dc * sf and the gate product), each <= 2^-24 of the magnitudes
    involved, and is carried with the factor sf <= 1 over at most S steps (4 S u).

    At L = 64 the dot product is the K = 256 FFMA dot of r2d2_lstm_bwd_kernel (FFMA_DOT).  At L = 256 / 512 it is the
    cluster sum: every term passes through n = r2d2_bwd_terms(L) roundings, so |err dh| <= gamma_n (|dhout| +
    sum |dz_{t+1}| |W_h|) per element.  Relative to the block's largest value that is gamma_n times the ratio of the
    terms' magnitude to |dh|; the bar allows a ratio of 2 (the carry adds the share of the later steps' dh errors that
    the forget gates pass on).  The o block, which has no carry, checks the same sum per element without that
    allowance, so a wrong partial cannot hide behind it."""
    return (FFMA_DOT if L == R2L else 2 * gamma(r2d2_bwd_terms(L))) + 4 * S * U


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
def R2D2_BUFFERS(L=R2L):
    """The R2D2 step's buffers at lstm_size ``L`` (as APEX_BUFFERS)."""
    return {
        "a1": ("M", (20, 20, 32)), "a2": ("M", (9, 9, 64)), "a3": ("M", (FLAT,)),
        "e1": ("A", (256,)), "emb": ("A", (256,)),
        "zx": ("M", (4 * L,)), "gates": ("M", (4 * L,)), "tc": ("M", (L,)), "hout": ("M", (L,)),
        "hin": ("M", (L,)), "cin": ("M", (L,)), "q1": ("M", (R2H,)), "q": ("MA", ()),
        "dq": ("M", (32,)), "dmean": ("M", (32,)), "dq1": ("M", (R2H,)), "dhout": ("M", (L,)), "dz": ("M", (4 * L,)),
        "da3": ("M", (FLAT,)), "du": ("M", (256,)), "da2": ("M", (9, 9, 64)), "da1": ("M", (20, 20, 32)),
    }


# the buffers an R2D2 td_error call writes (the main scope's forward)
R2D2_FWD_BUFFERS = ("a1", "a2", "a3", "e1", "emb", "zx", "gates", "tc", "hout", "hin", "cin", "q1", "q")


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


def _gates(z, L=R2L):
    i, j, f, o = (z[:, k * L:(k + 1) * L] for k in range(4))
    return np.concatenate([1 / (1 + np.exp(-i)), np.tanh(j), 1 / (1 + np.exp(-(f + 1.0))), 1 / (1 + np.exp(-o))], 1)


def r2d2_references(buf, p, batch, B, S, A, L=R2L, backward=True):
    """{output: float64 reference} of the R2D2 main-scope forward (trunk, lstm_x_fwd, the recurrence step by step from
    the kernel's stored state, q1, q) and the whole backward, each from the GPU buffers its kernel read.  The TD kernel
    is ``r2d2_td``.  Adds ``z`` (the recurrence's pre-activation, for bounds and regime checks) and ``cnext``: the
    reference c_t * (1 - done_t) of every row but the last step, which the next step's ``cin`` must hold.  At L > 64
    also ``zmag`` = |zx| + |b| + |h_in| |W_h| and ``dhmag`` = |dhout| + (1 - done) |dz_{t+1}| |W_h|^T, the magnitudes
    of the two cluster sums (r2d2_recurrence_bounds).  ``backward`` False: the forward only (a td_error call)."""
    inp = r2d2_inputs(batch)
    M = B * S
    P = _P(p)
    W = {k: _np(v) for k, v in P.items()}
    if backward:
        ref = lp.trunk_references(buf, P, inp["x"], inp["pa"], A, M)
    else:
        ref = lp.trunk_forward_references(buf, P, inp["x"], A)
    xcat = np.concatenate([buf["a3"], buf["emb"][inp["pa"]]], axis=1)
    Wx, Wh = W["lstm.w"][:XCAT], W["lstm.w"][XCAT:]
    ref["zx"] = xcat @ Wx
    # ---- recurrence, one step at a time from the stored state ----------------------------------------------------------
    z = buf["zx"] + W["lstm.b"] + buf["hin"] @ Wh
    g = _gates(z, L)
    si, tj, sf, so = (g[:, k * L:(k + 1) * L] for k in range(4))
    c = sf * buf["cin"] + si * tj
    ref["z"], ref["gates"], ref["c"] = z, g, c
    if L != R2L:
        ref["zmag"] = np.abs(buf["zx"]) + np.abs(W["lstm.b"]) + np.abs(buf["hin"]) @ np.abs(Wh)
    ref["tc"] = np.tanh(c)
    ref["hout"] = so * ref["tc"]
    keep = (~inp["done"]).astype(np.float64).T.reshape(M, 1)           # time-major rows
    ref["cnext"] = (c * keep)[:M - B]
    # ---- head ------------------------------------------------------------------------------------------------------
    ref["q1"] = np.maximum(buf["hout"] @ W["q1.w"] + W["q1.b"], 0.0)
    ref["q"] = (buf["q1"] @ W["value.w"] + W["value.b"]) - (buf["q1"] @ W["mean.w"] + W["mean.b"])
    if not backward:
        return ref
    # ---- backward ---------------------------------------------------------------------------------------------------
    dxv, ref["value.w"], ref["value.b"] = _dense(buf["q1"], W["value.w"], W["value.b"], buf["dq"][:, :A])
    dxm, ref["mean.w"], ref["mean.b"] = _dense(buf["q1"], W["mean.w"], W["mean.b"], buf["dmean"][:, :1])
    ref["dq1"] = (dxv + dxm) * _mask(buf["q1"])
    ref["dhout"], ref["q1.w"], ref["q1.b"] = _dense(buf["hout"], W["q1.w"], W["q1.b"], buf["dq1"])
    # BPTT: dz_t from the GPU's dhout_t, its forward buffers and its own dz_{t+1}; only the dc carry is re-run
    gg = buf["gates"]
    gi, gj, gf, go = (gg[:, k * L:(k + 1) * L] for k in range(4))
    dz = np.zeros((M, 4 * L))
    carry = np.zeros((B, L))
    dhmag = np.abs(buf["dhout"])
    for t in range(S - 1, -1, -1):
        r = slice(t * B, (t + 1) * B)
        kt = keep[r]
        dh = buf["dhout"][r] + (kt * (buf["dz"][(t + 1) * B:(t + 2) * B] @ Wh.T) if t < S - 1 else 0.0)
        if L != R2L and t < S - 1:
            dhmag[r] += kt * (np.abs(buf["dz"][(t + 1) * B:(t + 2) * B]) @ np.abs(Wh).T)
        dc = kt * carry + dh * go[r] * (1 - buf["tc"][r] ** 2)
        dz[r] = np.concatenate([dc * gj[r] * gi[r] * (1 - gi[r]), dc * gi[r] * (1 - gj[r] ** 2),
                                dc * buf["cin"][r] * gf[r] * (1 - gf[r]), dh * buf["tc"][r] * go[r] * (1 - go[r])], 1)
        carry = dc * gf[r]
    ref["dz"] = dz
    if L != R2L:
        ref["dhmag"] = dhmag
    dx, ref["lstm.w"], ref["lstm.b"] = _dense(np.concatenate([xcat, buf["hin"]], 1), W["lstm.w"], W["lstm.b"], buf["dz"])
    ref["da3"] = dx[:, :FLAT] * _mask(buf["a3"])
    ref["du"] = dx[:, FLAT:XCAT]
    return ref


def r2d2_recurrence_bounds(ref, cin, buf=None, L=R2L):
    """Per-element bounds of gates / tc / hout / cnext: ``layer_parity.lstm_bounds`` with the K = 64 FFMA dot product
    h_in W_h (and the add of zx and the bias) as the pre-activation bar; tc = tanh(c) carries c's bound with its
    derivative.

    At L > 64 the pre-activation is bounded per element from the cluster kernel's summation order,
    gamma_n (|zx| + |b| + sum |h| |W_h|) with n = r2d2_fwd_terms(L), and passed to lstm_bounds as its ``dz``.  The
    same order bounds the BPTT's dh per element, gamma_n (|dhout| + sum |dz_{t+1}| |W_h|) with n = r2d2_bwd_terms(L);
    the o block of dz, dh tc so (1 - so), does not see the dc carry and is held to that bound times its factor
    |tc so (1 - so)|, plus four roundings of its own (``dz/o``; needs ``buf``, the step's gates and tc)."""
    if L == R2L:
        b = lp.lstm_bounds(dict(z=ref["z"], gates=ref["gates"], c1=ref["c"]), cin, FFMA_DOT)
    else:
        b = lp.lstm_bounds(dict(z=ref["z"], gates=ref["gates"], c1=ref["c"]), cin, None,
                           dz=gamma(r2d2_fwd_terms(L)) * ref["zmag"])
    tc = ref["tc"]
    etc = (1 - tc ** 2) * b["c1"] + b["c1"] ** 2 + ELEM
    out = {"gates": b["gates"], "tc": etc, "hout": b["h1"], "cnext": b["c1"][:ref["cnext"].shape[0]]}
    if L != R2L and "dhmag" in ref:
        so, tcv = buf["gates"][:, 3 * L:], buf["tc"]
        out["dz/o"] = (np.abs(tcv * so * (1 - so)) * gamma(r2d2_bwd_terms(L)) * ref["dhmag"]
                       + gamma(4) * np.abs(ref["dz"][:, 3 * L:]) + TINY)
    return out


# ------------------------------------------------------------------------------------------------------------------
# metric
# ------------------------------------------------------------------------------------------------------------------
def r2d2_ntiles(L):
    """(label, columns) of the 256-wide N tiles of a [., 4L] LSTM GEMM output, each named by its gate: "f.n5"."""
    return [("%s.n%d" % ("ijfo"[n * R2_NTILE // L], n), slice(n * R2_NTILE, (n + 1) * R2_NTILE))
            for n in range(4 * L // R2_NTILE)]


def r2d2_ranks(L, gates="ijfo"):
    """(label, columns) of the cluster CTA ranks in a [., 4L] recurrence output (``gates`` = "": a [., L] one): rank r
    owns units [32 r, 32 r + 32) of every gate; labelled with the gate and the N tile that holds them, "j.n1.rank3"."""
    if not gates:
        return [("rank%d" % r, slice(32 * r, 32 * r + 32)) for r in range(L // 32)]
    return [("%s.n%d.rank%d" % (g, (k * L + 32 * r) // R2_NTILE, r), slice(k * L + 32 * r, k * L + 32 * r + 32))
            for k, g in enumerate("ijfo") if g in gates for r in range(L // 32)]


def r2d2_blocks(name, ref, L=R2L):
    """Natural sub-tensors of an R2D2 output: the i/j/f/o column blocks (L wide) of zx / gates / dz / lstm.w, the a3 /
    emb / h row segments of lstm.w; every other output as in ``layer_parity.blocks``.  At L > 64 the columns of zx and
    lstm.w are the 256-wide N tiles of their GEMMs, those of the recurrence's outputs (gates, tc, hout, dz) the CTA
    ranks of the cluster (``r2d2_ranks``); "dz/ijf" and "dz/o" are the carried and the uncarried blocks of dz."""
    rows = lp._row_tiles(ref.shape[0]) if ref.ndim else []
    if L == R2L:
        if name in ("zx", "gates", "dz"):
            return [("%s/r%d" % (g, s.start), (s, slice(k * R2L, (k + 1) * R2L)))
                    for k, g in enumerate("ijfo") for s in rows]
        if name == "lstm.w":
            segs = (("a3", 0, FLAT), ("emb", FLAT, XCAT), ("h", XCAT, XCAT + R2L))
            return [("%s.%s/r%d" % (sg, g, r0), (slice(r0, min(r0 + TILE, hi)), slice(k * R2L, (k + 1) * R2L)))
                    for sg, lo, hi in segs for r0 in range(lo, hi, TILE) for k, g in enumerate("ijfo")]
        if name == "lstm.b":
            return [(g, (slice(k * R2L, (k + 1) * R2L),)) for k, g in enumerate("ijfo")]
        return lp.blocks(name, ref)
    cols = {"zx": r2d2_ntiles(L), "gates": r2d2_ranks(L), "dz": r2d2_ranks(L), "dz/ijf": r2d2_ranks(L, "ijf"),
            "dz/o": [(lab, slice(c.start - 3 * L, c.stop - 3 * L)) for lab, c in r2d2_ranks(L, "o")],
            "tc": r2d2_ranks(L, ""), "hout": r2d2_ranks(L, ""), "cnext": r2d2_ranks(L, "")}
    if name in cols:
        return [("%s/r%d" % (lab, s.start), (s, c)) for lab, c in cols[name] for s in rows]
    if name == "lstm.w":
        segs = (("a3", 0, FLAT), ("emb", FLAT, XCAT), ("h", XCAT, XCAT + L))
        return [("%s.%s/r%d" % (sg, lab, r0), (slice(r0, min(r0 + TILE, hi)), c))
                for sg, lo, hi in segs for r0 in range(lo, hi, TILE) for lab, c in r2d2_ntiles(L)]
    if name == "lstm.b":
        return [(lab, (c,)) for lab, c in r2d2_ntiles(L)]
    return lp.blocks(name, ref)


def _worst_block(d, blocks):
    """The label of the block of ``blocks`` [(label, index)] that holds the largest value of ``d``."""
    worst, label = -1.0, ""
    for lab, idx in blocks:
        x = d[idx]
        if x.size and float(np.max(x)) > worst:
            worst, label = float(np.max(x)), lab
    return label


def bound_row(kernel, name, got, ref, bound, blocks=None):
    """A row held per element to ``bound`` (the ratio is reported; the per-tensor / block errors for information).
    ``blocks`` [(label, index)]: ``where`` names the one that holds the worst ratio."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    d = np.abs(got - ref)
    q = d / np.maximum(bound, TINY)
    ratio = float(np.max(q)) if d.size else 0.0
    if not np.all(np.isfinite(got)):
        ratio = float("inf")
    mx = float(np.max(np.abs(ref))) if ref.size else 0.0
    e = float(np.max(d)) / max(mx, 1e-30) if d.size else 0.0
    where = _worst_block(np.where(np.isfinite(q), q, np.inf), blocks) if blocks and d.size else ""
    return dict(kernel=kernel, tensor=name, err=e, block=e, where=where, bar="per-element bound", bound_ratio=ratio,
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


def r2d2_bars(S, L=R2L):
    """{output: bar}.  The six LSTM / q1 GEMMs (lstm_x_fwd, q1_fwd, q1_dgrad, q1_wgrad, lstm_wgrad, lstm_dgrad) keep the
    TF32 bar at every width.  Their 3xTF32 error follows the length of one CTA's accumulation chain (one split-K chunk),
    not the whole K: at the benchmark shape lstm_x_fwd's chunk is 256 / 848 / 1696 at L = 64 / 256 / 512 and zx
    measured 6.5e-6 at 256 and 1.2e-5 at 512; lstm_dgrad runs K = 4L unsplit and measured 6.7e-6 at 256 and 1.9e-5 at
    512 (one H100 80GB HBM3, 700 W).  The last is the closest any R2D2 GEMM comes to its bar."""
    b = {k: TF32 for k in R2D2_KERNEL}
    b.update(TRUNK_BAR)
    b.update(q=FFMA_DOT, dq1=FFMA_DOT, dz=r2d2_bptt_bar(S, L))
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


def _r2d2_recurrence_rows(got, ref, buf, inp, B, S, L):
    """The recurrence forward's per-element rows and its exact state hand-over: (h0, c0) at step 0, and
    hin[t+1] = hout_t (1 - done_t) (at L > 64 the distributed-shared-memory store to every rank)."""
    M = B * S
    eb = r2d2_recurrence_bounds(ref, buf["cin"], buf, L)
    rows = []
    for k in ("gates", "tc", "hout", "cnext"):
        blk = None if L == R2L else r2d2_blocks(k, ref[k], L)
        rows.append(bound_row("r2d2_lstm_fwd", k, got[k], ref[k], eb[k], blk))
    keep = (~inp["done"]).astype(np.float64).T.reshape(M, 1)
    rows.append(exact_row("r2d2_lstm_fwd", "hin[0]", buf["hin"][:B], inp["h0"]))
    rows.append(exact_row("r2d2_lstm_fwd", "cin[0]", buf["cin"][:B], inp["c0"]))
    rows.append(exact_row("r2d2_lstm_fwd", "hin[t+1]", buf["hin"][B:], (buf["hout"] * keep)[:M - B]))
    return rows, eb


def check_r2d2(buf, grads, p, batch, taps, out, B, S, bi, A, gamma, L=R2L):
    """Rows of every checked output of one R2D2 step (see check_apex), the exact checks of the recurrence's state
    hand-over and of the gradient rows outside the loss window included.  At L > 64 the dz row holds the i / j / f
    blocks to r2d2_bptt_bar and a ``dz/o`` row the o block per element (r2d2_recurrence_bounds): one row more."""
    M = B * S
    ref = r2d2_references(buf, p, batch, B, S, A, L)
    inp = r2d2_inputs(batch)
    got = dict(buf)
    got.update(grads)
    got["cnext"] = buf["cin"][B:]
    bar = r2d2_bars(S, L)
    blocks = functools.partial(r2d2_blocks, L=L)
    rows = []
    for k in R2D2_KERNEL:
        if k == "dz" and L != R2L:
            rows.append(bar_row(R2D2_KERNEL[k], "dz/ijf", got[k][:, :3 * L], ref[k][:, :3 * L], bar[k], blocks))
        else:
            rows.append(bar_row(R2D2_KERNEL[k], k, got[k], ref[k], bar[k], blocks))
    rec, eb = _r2d2_recurrence_rows(got, ref, buf, inp, B, S, L)
    rows += rec
    if L != R2L:
        rows.append(bound_row(R2D2_KERNEL["dz"], "dz/o", got["dz"][:, 3 * L:], ref["dz"][:, 3 * L:], eb["dz/o"],
                              r2d2_blocks("dz/o", ref["dz"][:, 3 * L:], L)))
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


R2D2_FWD_KERNEL = {k: R2D2_KERNEL[k] for k in ("a1", "a2", "a3", "e1", "emb", "zx", "q1", "q")}


def check_r2d2_forward(buf, p, batch, B, S, A, L=R2L):
    """Rows of the main scope's forward of a td_error call over B sequences (the kernels of ``R2D2_FWD_KERNEL``, the
    recurrence's per-element rows and its exact state hand-over), as check_r2d2."""
    ref = r2d2_references(buf, p, batch, B, S, A, L, backward=False)
    got = dict(buf)
    got["cnext"] = buf["cin"][B:]
    bar = r2d2_bars(S, L)
    blocks = functools.partial(r2d2_blocks, L=L)
    rows = [bar_row(R2D2_FWD_KERNEL[k], k, got[k], ref[k], bar[k], blocks) for k in R2D2_FWD_KERNEL]
    rows += _r2d2_recurrence_rows(got, ref, buf, r2d2_inputs(batch), B, S, L)[0]
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


def scale_lstm(L=R2L):
    """The saturated regime's factor on lstm.w at width L: SCALE_LSTM at 64, rescaled so that the h half of the
    pre-activation keeps its spread.  Its terms are Glorot-uniform weights of limit sqrt(6 / (3392 + 5 L)) (lstm.w is
    [3392 + L, 4L]) over a sum of L units, so its standard deviation goes as limit * sqrt(L): 33.7 at 256, 26.9 at 512.
    (The [a3 | emb] half then keeps sqrt(64 / L) of its spread at 64: 0.5 and 0.35.)  Measured with the
    oracle at init over four 80-step sequences: |z| > 4 for 48 % of the gates at 64, 35 % at 256 and 36 % at 512."""
    lim = lambda n: math.sqrt(6.0 / (XCAT + 5 * n))
    return SCALE_LSTM * lim(R2L) / lim(L) * math.sqrt(R2L / L) if L != R2L else SCALE_LSTM


def run_r2d2_case(mode, B, S, bi, A, C, regime, seed=2468, L=R2L):
    """One step of a fresh R2D2 learner of lstm_size ``L`` in ``regime``; returns (rows, facts) as
    layer_parity.run_case."""
    import r2d2_parity
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET, NativeR2D2Learner
    kw = dict(num_action=A, lstm_size=L, input_shape=(84, 84, C))
    params = rt.init_params(0, torch.float32, **kw)
    target = rt.init_params(1, torch.float32, **kw)
    if regime == "saturated":
        params["lstm.w"] = params["lstm.w"] * scale_lstm(L)
    if regime == "large_returns":
        target["value.b"] = torch.full((A,), BIG_RETURN, dtype=torch.float32)
    if regime == "ties":            # two identical value columns, raised above the others: exact ties at the maximum
        params["value.w"][:, 1] = params["value.w"][:, 0]
        params["value.b"][:2] = 1.0
    done_rate, done_ends = (0.3, True) if regime == "done_heavy" else (None, False)
    lr = TRAIN_LR if regime == "trained" else rt.LR
    eng = NativeR2D2Learner(batch=B, seq_len=S, burn_in=bi, num_action=A, lstm_size=L, input_shape=(84, 84, C),
                            math_mode=mode, learning_rate=lr)

    def stage(s):
        b = r2d2_parity.make_batch(B, S, A, C, s, done_rate, done_ends, L=L)
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
        buf = read_buffers(eng, R2D2_BUFFERS(L), B * S, B * S, A)
        grads = {k: v.numpy() for k, v in rt.unflatten_params(eng.get_grads(), torch.float64, **kw).items()}
    finally:
        eng.close()
    rows, ref = check_r2d2(buf, grads, p, batch, taps, dict(o, td=td), B, S, bi, A,
                           float(np.float32(rt.DEFAULT_CFG["discount_factor"])), L)
    facts["finite"] = bool(all(np.all(np.isfinite(v)) for v in list(buf.values()) + list(grads.values())))
    facts["z_abs_gt4"] = float(np.mean(np.abs(ref["z"]) > 4))
    facts["c_abs_max"] = float(np.abs(ref["c"]).max())
    facts["done_rate"] = float(np.mean(batch["done"]))
    facts["done_ends"] = bool(batch["done"][:, 0].all() and batch["done"][:, -1].all())
    facts["target_abs_max"] = float(np.abs(taps["target_q"]).max())        # what h^-1 reads
    mq = taps["main_q"][:, bi + 1:]
    facts["tie_rows"] = int(np.sum(mq.max(2) == np.sort(mq, 2)[..., -2]))
    return rows, facts


def run_r2d2_td_error_case(mode, ns, S, bi, A, C, L, seed=1357):
    """td_error calls over n = each of ``ns`` sequences on one fresh R2D2 learner of batch max(ns) at width L; after
    each call, the rows of its main-scope forward (check_r2d2_forward, from the buffers of that call).
    -> {n: rows}."""
    import r2d2_parity
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET, NativeR2D2Learner
    kw = dict(num_action=A, lstm_size=L, input_shape=(84, 84, C))
    eng = NativeR2D2Learner(batch=max(ns), seq_len=S, burn_in=bi, num_action=A, lstm_size=L, input_shape=(84, 84, C),
                            math_mode=mode)
    table = R2D2_BUFFERS(L)
    out = {}
    try:
        eng.set_params(rt.flatten_params(rt.init_params(0, torch.float32, **kw)), MAIN)
        eng.set_params(rt.flatten_params(rt.init_params(1, torch.float32, **kw)), TARGET)
        p = rt.unflatten_params(eng.get_params(), torch.float64, **kw)
        for n in ns:
            b = r2d2_parity.make_batch(n, S, A, C, seed + n, 0.3, True, L=L)
            eng.td_error(b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"],
                         b["done"])
            buf = read_buffers(eng, {k: table[k] for k in R2D2_FWD_BUFFERS}, n * S, n * S, A)
            out[n] = check_r2d2_forward(buf, p, b, n, S, A, L)[0]
    finally:
        eng.close()
    return out


def launch_facts():
    """The split-K counts the library plans (drl_debug_apex_launch_plan / drl_debug_r2d2_launch_plan) for a shape:
    ``apex(B, mode)`` -> dict(heads_l1_fwd, conv1_wgrad, conv2_wgrad, conv3_wgrad); ``r2d2(B, S, C, mode, L)`` -> the
    same with lstm_x_fwd for heads_l1_fwd, and R: the sequences per cluster pass of the recurrence (0 at L = 64)."""
    import ctypes
    from distributed_reinforcement_learning_b200 import _native as N

    def apex(B, mode):
        out = (ctypes.c_int32 * 4)()
        N.check(N.lib.drl_debug_apex_launch_plan(B, mode, out))
        return dict(heads_l1_fwd=out[0], conv1_wgrad=out[1], conv2_wgrad=out[2], conv3_wgrad=out[3])

    def r2d2(B, S, C, mode, L=R2L):
        out = (ctypes.c_int32 * 5)()
        N.check(N.lib.drl_debug_r2d2_launch_plan(B, S, C, mode, L, out))
        return dict(lstm_x_fwd=out[0], conv1_wgrad=out[1], conv2_wgrad=out[2], conv3_wgrad=out[3], R=out[4])
    return apex, r2d2
