"""Per-kernel float64 references of the IMPALA learner step, fed from the step's own buffers.

``parity.compare_step`` judges the whole step against the float64 oracle, so the rounding of every kernel upstream of a
tensor adds to that tensor's error.  Here each kernel is judged only from the buffers it read: ``references`` takes the
device buffers of one step (``read_step``), the parameters the step ran with and the staged batch, and returns for every
kernel output the float64 value the kernel should have written, computed with the oracle's layer functions
(``oracle.impala_torch``) and torch autograd (a backward kernel's upstream gradient is the GPU's own buffer, passed as
``grad_outputs``).

Device conventions (csrc/learner.cu, csrc/layers.cu):
  * activation rows are time-major, m = t*B + b; the batch (frames, h0, c0, previous action) is staged batch-major;
  * backward buffers hold the first Mb = B*(T-2) rows (the steps t <= T-3 that receive gradient);
  * d* buffers are gradients with respect to the pre-ReLU value, i.e. they carry the mask of the GPU's own activation;
  * hid1 / hid2 / dhid2 / dhid1 / dh_part stack the actor half on top of the critic half;
  * dlogits and dv have 32 columns (dv: column 0);
  * gates = [sigmoid(i) | tanh(j) | sigmoid(f + 1) | sigmoid(o)] (csrc/elementwise.cu, lstm_gates_forward_kernel);
  * frames are divided by 255 in float32 (agent/impala.py:133 feeds float32).

Metrics (``errors``): per tensor max|gpu - ref| / max|ref| (= ``parity.rel_err``); per block
max|gpu - ref|_block / max(max|ref|_block, 1e-2 max|ref|_tensor) over the natural sub-tensors: 128-row tiles of the
GEMM row dimension, the i/j/f/o column blocks of gates / dz / lstm.w, the a3 / emb / h row segments of lstm.w, the
actor / critic halves.  The block error catches a wrong partial tile or segment whose values are small next to the
tensor's maximum.
"""
import numpy as np
import torch

from oracle import impala_torch as it
from oracle import synthetic

L = 256
G4 = 4 * L
FLAT = 7 * 7 * 64
XK = FLAT + 256 + L
TILE = 128
BLOCK_FLOOR = 1e-2

# buffer name -> per-row shape (rows: "M" forward rows, "Mb" backward rows, "A" actions); "2" = actor/critic halves
BUFFERS = {
    "a1": ("M", (20, 20, 32)), "a2": ("M", (9, 9, 64)), "a3": ("M", (FLAT,)),
    "e1": ("A", (256,)), "emb": ("A", (256,)),
    "gates": ("M", (G4,)), "h1": ("M", (L,)), "c1": ("M", (L,)),
    "hid1": ("2M", (256,)), "hid2": ("2M", (256,)),
    "logits": ("MA", ()), "policy": ("MA", ()), "value": ("M", ()),
    "dlogits": ("Mb", (32,)), "dv": ("Mb", (32,)),
    "dhid2": ("2Mb", (256,)), "dhid1": ("2Mb", (256,)), "dh_part": ("2Mb", (L,)),
    "dz": ("Mb", (G4,)), "da3": ("Mb", (FLAT,)), "du": ("Mb", (256,)),
    "da2": ("Mb", (9, 9, 64)), "da1": ("Mb", (20, 20, 32)),
}


def time_major(x_bt):
    """[B, T, ...] -> [T*B, ...] (rows m = t*B + b)."""
    x = np.asarray(x_bt)
    return np.swapaxes(x, 0, 1).reshape((x.shape[0] * x.shape[1],) + x.shape[2:])


def read_step(eng, B, T, A):
    """Every intermediate buffer of the step the engine just ran, as float64 arrays in device layout."""
    M, Mb = B * T, B * (T - 2)
    out = {}
    for name, (rows, shp) in BUFFERS.items():
        if rows == "MA":
            n, shape = M * A, (M, A)
        elif rows == "A":
            n, shape = A * int(np.prod(shp)), (A,) + shp
        else:
            r = {"M": M, "Mb": Mb, "2M": 2 * M, "2Mb": 2 * Mb}[rows]
            n, shape = r * int(np.prod(shp)), ((2, r // 2) if rows.startswith("2") else (r,)) + shp
        out[name] = eng.read_buffer(name, n).astype(np.float64).reshape(shape)
    return out


def device_inputs(batch):
    """The staged batch in device row order: frames / 255 (float32 divide), previous action, h0, c0."""
    x = (time_major(batch["state"]).astype(np.float32) / np.float32(255.0)).astype(np.float64)
    return dict(x=x, pa=time_major(batch["previous_action"]).astype(np.int64),
                h0=time_major(batch["initial_h"]).astype(np.float64), c0=time_major(batch["initial_c"]).astype(np.float64))


def _t(x, grad=False):
    t = torch.as_tensor(np.asarray(x, np.float64))
    return t.clone().requires_grad_(True) if grad else t


def _np(t):
    return t.detach().numpy()


def _mask(x):
    return (np.asarray(x) > 0).astype(np.float64)


def _dense(x, w, b, dy):
    """(dx, dw, db) of y = x @ w + b for the upstream gradient dy (the last line of it.fully_connected)."""
    xt, wt, bt = _t(x, True), _t(w, True), _t(b, True)
    y = xt @ wt + bt
    return tuple(_np(g) for g in torch.autograd.grad(y, (xt, wt, bt), _t(dy)))


def _conv_grads(x, w, b, stride, dy):
    """(dx, dw, db) of it._conv2d_tf(x, w, b, stride) for the upstream gradient dy (NHWC, HWIO)."""
    xt, wt, bt = _t(x, True), _t(w, True), _t(b, True)
    y = it._conv2d_tf(xt, wt, bt, stride)
    return tuple(_np(g) for g in torch.autograd.grad(y, (xt, wt, bt), _t(dy)))


def vtrace_grads(policy, value, batch, cfg, B, T, A):
    """dL/dlogits and dL/dvalue of the total loss (``it.loss_terms``, agent/impala.py:45-93) at the given time-major
    policy / value rows.  The fused V-trace kernel reads the policy, not the logits: logits = log(policy) makes
    softmax(logits) = policy, so autograd through softmax gives the kernel's p * (g - sum p g)."""
    lg = _t(np.log(np.asarray(policy).reshape(T, B, A)).swapaxes(0, 1), True)
    val = _t(np.asarray(value).reshape(T, B).swapaxes(0, 1), True)
    pol = torch.softmax(lg, dim=2)
    c = dict(it.DEFAULT_CFG)
    c.update(cfg)
    prep = it.loss_inputs(batch["reward"], batch["action"], batch["done"], batch["behavior_policy"], torch.float64)
    fp, mp, lp = it.split_data(pol)
    fv, mv, lv = it.split_data(val)
    total = it.loss_terms(c, prep, fp, fv, mp, mv, lp, lv)["total_loss"]
    glg, gv = torch.autograd.grad(total, (lg, val))
    Mb = B * (T - 2)
    return time_major(_np(glg))[:Mb], time_major(_np(gv))[:Mb]


def gates_backward(dh, gates, c1, c0):
    """dz from dh and the cell's own gate values: autograd of c = sf*c0 + si*tj, h = so*tanh(c) with respect to the
    four gate values, times the derivative of each gate's nonlinearity written in its output (s(1-s), 1-t^2) -- the
    lstm_gates_bwd kernel's formula, evaluated in float64 from the values the forward kernel stored."""
    g = _t(gates, True)
    si, tj, sf, so = torch.chunk(g, 4, dim=1)
    c = sf * _t(c0) + si * tj
    c = c + (_t(c1) - c).detach()      # the value the kernel read (c1, rounded to float32), the derivative of the sum
    h = so * torch.tanh(c)
    (dg,) = torch.autograd.grad(h, (g,), _t(dh))
    gv = np.asarray(gates, np.float64)
    deriv = np.concatenate([gv[:, :L] * (1 - gv[:, :L]), 1 - gv[:, L:2 * L] ** 2,
                            gv[:, 2 * L:3 * L] * (1 - gv[:, 2 * L:3 * L]), gv[:, 3 * L:] * (1 - gv[:, 3 * L:])], axis=1)
    return _np(dg) * deriv


def references(buf, p, batch, cfg, B, T, A):
    """{output name: float64 reference}, each computed from the GPU buffers its kernel read.
    ``p``: the parameters the step ran with (float64 torch tensors by name); ``batch``: the staged batch."""
    Mb = B * (T - 2)
    inp = device_inputs(batch)
    P = {k: v.detach().to(torch.float64) for k, v in p.items()}
    ref = trunk_references(buf, P, inp["x"], inp["pa"], A, Mb)
    with torch.no_grad():
        # ---- forward -----------------------------------------------------------------------------------------
        x = torch.cat([_t(buf["a3"]), _t(buf["emb"])[torch.from_numpy(inp["pa"])]], dim=1)
        h0, c0 = _t(inp["h0"]), _t(inp["c0"])
        z = torch.cat([x, h0], dim=1) @ P["lstm.w"] + P["lstm.b"]
        i, j, f, o = torch.chunk(z, 4, dim=1)
        ref["z"] = _np(z)       # not a buffer: the pre-activation the lstm_fwd GEMM produced (bars, regime checks)
        ref["gates"] = _np(torch.cat([torch.sigmoid(i), torch.tanh(j), torch.sigmoid(f + 1.0), torch.sigmoid(o)], 1))
        h1, c1, _ = it.lstm(P, x, h0, c0)
        ref["h1"], ref["c1"] = _np(h1), _np(c1)
        hid1, hid2 = [], []
        for zi, pre in enumerate(("actor", "critic")):
            hid1.append(torch.relu(_t(buf["h1"]) @ P[pre + "1.w"] + P[pre + "1.b"]))
            hid2.append(torch.relu(_t(buf["hid1"][zi]) @ P[pre + "2.w"] + P[pre + "2.b"]))
        ref["hid1"], ref["hid2"] = _np(torch.stack(hid1)), _np(torch.stack(hid2))
        ref["logits"] = _np(_t(buf["hid2"][0]) @ P["actor3.w"] + P["actor3.b"])
        ref["policy"] = _np(torch.softmax(_t(buf["logits"]), dim=1))   # same kernel: softmax of the logits it stored
        ref["value"] = _np(_t(buf["hid2"][1]) @ P["critic3.w"] + P["critic3.b"])[:, 0]
    # ---- V-trace + loss gradient --------------------------------------------------------------------------------
    dl, dv = vtrace_grads(buf["policy"], buf["value"], batch, cfg, B, T, A)
    ref["dlogits"], ref["dv"] = dl, dv
    # ---- heads backward ----------------------------------------------------------------------------------------
    gdl, gdv = buf["dlogits"][:, :A], buf["dv"][:, :1]
    W = {k: _np(v) for k, v in P.items()}
    hid1_b, hid2_b = buf["hid1"][:, :Mb], buf["hid2"][:, :Mb]
    dxa, ref["actor3.w"], ref["actor3.b"] = _dense(hid2_b[0], W["actor3.w"], W["actor3.b"], gdl)
    dxc, ref["critic3.w"], ref["critic3.b"] = _dense(hid2_b[1], W["critic3.w"], W["critic3.b"], gdv)
    ref["dhid2"] = np.stack([dxa, dxc]) * _mask(hid2_b)
    dh1, dhp = [], []
    for zi, pre in enumerate(("actor", "critic")):
        dx, ref[pre + "2.w"], ref[pre + "2.b"] = _dense(hid1_b[zi], W[pre + "2.w"], W[pre + "2.b"], buf["dhid2"][zi])
        dh1.append(dx * _mask(hid1_b[zi]))
        dx, ref[pre + "1.w"], ref[pre + "1.b"] = _dense(buf["h1"][:Mb], W[pre + "1.w"], W[pre + "1.b"],
                                                        buf["dhid1"][zi])
        dhp.append(dx)
    ref["dhid1"], ref["dh_part"] = np.stack(dh1), np.stack(dhp)
    # ---- LSTM cell and layer -----------------------------------------------------------------------------------
    ref["dz"] = gates_backward(buf["dh_part"][0] + buf["dh_part"][1], buf["gates"][:Mb], buf["c1"][:Mb],
                               inp["c0"][:Mb])
    xb = np.concatenate([buf["a3"][:Mb], buf["emb"][inp["pa"][:Mb]], inp["h0"][:Mb]], axis=1)
    dx, ref["lstm.w"], ref["lstm.b"] = _dense(xb, W["lstm.w"], W["lstm.b"], buf["dz"])
    ref["da3"] = dx[:, :FLAT] * _mask(buf["a3"][:Mb])
    ref["du"] = dx[:, FLAT:FLAT + 256]
    return ref


def trunk_forward_references(buf, P, x, A, emb_key="emb"):
    """The forward half of ``trunk_references`` (also the policy engines' trunk): conv1 from the frames ``x`` / 255,
    conv2 / conv3 from the GPU's a1 / a2, the embedding's first layer from the parameters and its table from the GPU's
    e1.  ``emb_key``: the name of the table (the learners' "emb", the policy engines' "table")."""
    M = x.shape[0]
    ref = {}
    with torch.no_grad():
        ref["a1"] = _np(torch.relu(it._conv2d_tf(_t(x), P["conv1.w"], P["conv1.b"], 4)))
        ref["a2"] = _np(torch.relu(it._conv2d_tf(_t(buf["a1"]), P["conv2.w"], P["conv2.b"], 2)))
        ref["a3"] = _np(torch.relu(it._conv2d_tf(_t(buf["a2"]), P["conv3.w"], P["conv3.b"], 1))).reshape(M, FLAT)
        acts = torch.arange(A)
        ref["e1"] = _np(torch.relu(torch.nn.functional.one_hot(acts, A).to(torch.float64) @ P["emb1.w"] + P["emb1.b"]))
        ref[emb_key] = _np(torch.relu(_t(buf["e1"]) @ P["emb2.w"] + P["emb2.b"]))
    return ref


def trunk_references(buf, P, x, pa, A, Mb):
    """References of the conv trunk and the action embedding that the IMPALA, Ape-X / A3C and R2D2 learners share
    (csrc/layer_defs.cuh): conv1-3 and the embedding forward from the GPU's own inputs to each layer, the embedding
    weight gradients from the GPU's ``du`` at the GPU's e1 / table masks, the conv data and weight gradients from the
    GPU's ``da3`` over the first ``Mb`` rows.  ``P``: float64 parameters by name; ``x``: the frames / 255 in device row
    order ([M, 84, 84, C], any channel count C); ``pa``: the previous action of every device row."""
    ref = trunk_forward_references(buf, P, x, A)
    W = {k: _np(v) for k, v in P.items()}
    # ---- action embedding weight gradients (at the GPU's e1 / table masks) ---------------------------------------
    pe = {k: _t(W[k], True) for k in ("emb1.w", "emb1.b", "emb2.w", "emb2.b")}
    masks = {"e1": torch.from_numpy(buf["e1"] > 0), "emb": torch.from_numpy(buf["emb"] > 0)}
    with it.activation_pattern(masks):
        rows = it.action_embedding(pe, torch.from_numpy(np.asarray(pa)[:Mb]), A)
    grads = torch.autograd.grad(rows, list(pe.values()), _t(buf["du"]))
    ref.update({k: _np(g) for k, g in zip(pe, grads)})
    # ---- convolutions: data gradients from the GPU's upstream gradient, weight gradients ---------------------------
    a2b, a1b = buf["a2"][:Mb], buf["a1"][:Mb]
    da3 = buf["da3"].reshape(Mb, 7, 7, 64)
    dx, ref["conv3.w"], ref["conv3.b"] = _conv_grads(a2b, W["conv3.w"], W["conv3.b"], 1, da3)
    ref["da2"] = dx * _mask(a2b)
    dx, ref["conv2.w"], ref["conv2.b"] = _conv_grads(a1b, W["conv2.w"], W["conv2.b"], 2, buf["da2"])
    ref["da1"] = dx * _mask(a1b)
    _, ref["conv1.w"], ref["conv1.b"] = _conv_grads(x[:Mb], W["conv1.w"], W["conv1.b"], 4, buf["da1"])
    return ref


def conv1_bound(x_u8_over_255, w, b):
    """Per-element error bound of the math-mode-5 conv1 forward (conv1_tma.cuh, fp16 split weights; gemm_umma16.cuh
    header): each weight is carried as hi + lo in fp16 with |w - hi - lo| <= max(2^-22 |w|, 2^-25) (2^-25: half the
    smallest fp16 subnormal, where the lo plane underflows), the frames are exact; plus the fp32 accumulation of the
    products (2^-20 of sum |x w|: 16 K-steps of K = 16 and the hi + lo add, with room), the bias add and the rounding
    of the result (2^-23 |z|)."""
    xt = _t(x_u8_over_255)
    e = torch.clamp(torch.abs(w) * 2.0 ** -22, min=2.0 ** -25)
    zero = torch.zeros_like(b)
    split = it._conv2d_tf(xt, e, zero, 4)
    acc = it._conv2d_tf(xt, torch.abs(w), zero, 4) * 2.0 ** -20
    z = it._conv2d_tf(xt, w, b, 4)
    return _np(split + acc + (torch.abs(b) + torch.abs(z)) * 2.0 ** -23)


# ------------------------------------------------------------------------------------------------------------------
# metric
# ------------------------------------------------------------------------------------------------------------------
def _row_tiles(n, tile=TILE):
    return [slice(r, min(r + tile, n)) for r in range(0, n, tile)]


def blocks(name, ref):
    """Natural sub-tensors of one output, as (label, index) pairs over ``ref`` in the GEMM's 2-D view."""
    if name in ("hid1", "hid2", "dhid2", "dhid1", "dh_part"):       # [2, rows, 256]: halves x row tiles
        return [("%s/r%d" % (h, s.start), (zi, s, slice(None)))
                for zi, h in enumerate(("actor", "critic")) for s in _row_tiles(ref.shape[1])]
    if name in ("gates", "dz"):
        return [("%s/r%d" % (g, s.start), (s, slice(k * L, (k + 1) * L)))
                for k, g in enumerate("ijfo") for s in _row_tiles(ref.shape[0])]
    if name == "lstm.w":
        segs = (("a3", 0, FLAT), ("emb", FLAT, FLAT + 256), ("h", FLAT + 256, XK))
        return [("%s.%s/r%d" % (sg, g, r0), (slice(r0, min(r0 + TILE, hi)), slice(k * L, (k + 1) * L)))
                for sg, lo, hi in segs for r0 in range(lo, hi, TILE) for k, g in enumerate("ijfo")]
    if name == "lstm.b":
        return [(g, (slice(k * L, (k + 1) * L),)) for k, g in enumerate("ijfo")]
    if ref.ndim == 4 and name.startswith("conv"):                     # HWIO weight: rows = (ky, kx, ci)
        n = ref.shape[0] * ref.shape[1] * ref.shape[2]
        return [("r%d" % s.start, s) for s in _row_tiles(n)]
    if name in ("a1", "a2", "da1", "da2"):                            # rows = pixels
        n = ref.shape[0] * ref.shape[1] * ref.shape[2]
        return [("px%d" % s.start, s) for s in _row_tiles(n)]
    return [("r%d" % s.start, s) for s in _row_tiles(ref.shape[0])]


def _view2d(name, x):
    if x.ndim == 4 and (name.startswith("conv") or name in ("a1", "a2", "da1", "da2")):
        return x.reshape(-1, x.shape[-1])
    return x


def errors(name, got, ref, blocks_of=None):
    """(per-tensor error, worst block error, worst block label); ``blocks_of``: the block function (default
    ``blocks``)."""
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    if not np.all(np.isfinite(got)):
        return float("inf"), float("inf"), "non-finite"
    d = np.abs(got - ref)
    mx = float(np.max(np.abs(ref))) if ref.size else 0.0
    tens = float(np.max(d)) / max(mx, 1e-30) if ref.size else 0.0
    g2, r2 = _view2d(name, d), _view2d(name, np.abs(ref))
    worst, label = 0.0, ""
    for lab, idx in (blocks_of or blocks)(name, ref):
        db, rb = g2[idx], r2[idx]
        if db.size == 0:
            continue
        e = float(np.max(db)) / max(float(np.max(rb)), BLOCK_FLOOR * mx, 1e-30)
        if e > worst:
            worst, label = e, lab
    return tens, worst, label


def gpu_outputs(buf, grads, A):
    """The GPU's value of every output ``references`` computes: buffers (dlogits / dv cut to their live columns)
    and the parameter gradients by name."""
    out = {k: v for k, v in buf.items()}
    out["dlogits"] = buf["dlogits"][:, :A]
    out["dv"] = buf["dv"][:, 0]
    out.update(grads)
    return out


def run_step(eng, batch, B, T, A):
    """Stage ``batch``, run one step; returns (buffers, parameter gradients by name, parameters the step ran with)."""
    p = it.unflatten_params(eng.get_params(), torch.float64, num_action=A)
    eng.stage(0, *[batch[k] for k in synthetic.TRAIN_FIELDS])
    eng.step(0)
    buf = read_step(eng, B, T, A)
    g = it.unflatten_params(eng.get_grads(), torch.float64, num_action=A)
    return buf, {k: v.numpy() for k, v in g.items()}, p


# ------------------------------------------------------------------------------------------------------------------
# bars: each from the error model of the core that computes the output
# ------------------------------------------------------------------------------------------------------------------
# 16-bit split cores (gemm_umma16.cuh, math mode 5; bf16 hi + lo, A_lo*B_lo dropped): ~2^-16 per product, random sign ->
# 2e-5 of the largest output, 3e-5 once K >= 1024 (the bars test_gpu_umma16.py holds the same cores to).  3xTF32
# (gemm_umma.cuh) and FP32 FFMA contractions: 2e-5 (test_gpu_umma.py: 1e-5 at K <= 100, 2e-5 at K = 3648).  The small
# FFMA dot products of heads_out_fwd / heads_out_bwd (K = 256 / K = A): 1e-5.  Elementwise kernels whose reference
# reads the same float32 inputs (embedding layer 1, softmax of the stored logits, the LSTM gate backward): 1e-6, a few
# float32 roundings.  The fused V-trace kernel: 1e-5 (a scan of up to 32 float32 affine maps over logs and exps).
SPLIT16, SPLIT16_LONGK, TF32, FFMA_DOT, ELEM, VTRACE = 2e-5, 3e-5, 2e-5, 1e-5, 1e-6, 1e-5

KERNEL = {"a1": "conv1_fwd", "a2": "conv2_fwd", "a3": "conv3_fwd", "e1": "emb_fwd", "emb": "emb_fwd",
          "gates": "lstm_fwd+gates_fwd", "c1": "lstm_fwd+gates_fwd", "h1": "lstm_fwd+gates_fwd",
          "hid1": "heads_l1_fwd", "hid2": "heads_l2_fwd", "logits": "heads_out_fwd", "value": "heads_out_fwd",
          "policy": "heads_out_fwd", "dlogits": "vtrace_losses", "dv": "vtrace_losses", "dhid2": "heads_out_bwd",
          "dhid1": "heads_l2_dgrad", "dh_part": "heads_l1_dgrad", "dz": "lstm_gates_bwd", "da3": "lstm_dgrad",
          "du": "lstm_dgrad", "da2": "conv3_dgrad", "da1": "conv2_dgrad",
          "actor3.w": "actor3_wgrad", "actor3.b": "actor3_wgrad", "critic3.w": "critic3_wgrad",
          "critic3.b": "critic3_wgrad", "actor2.w": "heads_l2_wgrad", "actor2.b": "heads_l2_wgrad",
          "critic2.w": "heads_l2_wgrad", "critic2.b": "heads_l2_wgrad", "actor1.w": "heads_l1_wgrad",
          "actor1.b": "heads_l1_wgrad", "critic1.w": "heads_l1_wgrad", "critic1.b": "heads_l1_wgrad",
          "lstm.w": "lstm_wgrad", "lstm.b": "lstm_wgrad(bias reduce)", "emb1.w": "emb_bwd", "emb1.b": "emb_bwd",
          "emb2.w": "emb_bwd", "emb2.b": "emb_bwd", "conv3.w": "conv3_wgrad+reduce", "conv3.b": "conv3_wgrad+reduce",
          "conv2.w": "conv2_wgrad+reduce", "conv2.b": "conv2_wgrad+reduce", "conv1.w": "conv1_wgrad+reduce",
          "conv1.b": "conv1_wgrad+reduce"}


def bars(mode, B, T):
    """{output: bar} for one step of math mode ``mode`` (all outputs but the per-element ones: mode-5 a1, gates, c1,
    h1)."""
    Mb = B * (T - 2)
    m16 = mode == 5
    gemm = SPLIT16 if m16 else TF32
    longk = SPLIT16_LONGK if m16 else TF32
    b = {"a2": gemm, "a3": gemm, "e1": ELEM, "emb": FFMA_DOT, "hid1": gemm, "hid2": gemm,
         "logits": FFMA_DOT, "value": FFMA_DOT, "policy": ELEM, "dlogits": VTRACE, "dv": VTRACE, "dhid2": FFMA_DOT,
         "dhid1": gemm, "dh_part": gemm, "dz": ELEM, "da3": longk, "du": longk, "da2": gemm, "da1": gemm}
    if not m16:
        b["a1"] = TF32
    # gates / c1 / h1 (lstm_fwd + lstm_gates_fwd) are held per element to lstm_bounds, from the long-K bar on z
    # weight gradients: the head ones are FFMA (every mode); lstm.w is the bulk-fed 16-bit core in mode 5 (K = Mb); the
    # conv ones are 16-bit (mode 5: K = Mb * pixels >= 1024) or 3xTF32 / FFMA; the biases are fp32 column sums
    for k in KERNEL:
        if "." in k:
            b[k] = TF32
    if m16:
        b["lstm.w"] = SPLIT16_LONGK if Mb >= 1024 else SPLIT16
        for k in ("conv3.w", "conv3.b", "conv2.w", "conv2.b", "conv1.w", "conv1.b"):
            b[k] = SPLIT16_LONGK
    return b


def lstm_bounds(ref, c0, zbar, dz=None):
    """Per-element bounds of the gates, c1 and h1 the LSTM kernels wrote, from the error model of the contraction that
    produced the pre-activation z: an error of at most dz = zbar * max|z| per element (IMPALA's lstm_fwd, K = 3648: the
    long-K bar of its core; R2D2's recurrence: the K = 64 FFMA dot product; relative to max|z| like every GEMM bar
    here) or, when given, the per-element bound ``dz`` (the policy engines' split sum, tests/policy_layer_parity.py),
    carried through each nonlinearity by its derivative at the reference value
    (sigmoid: s(1-s), tanh: 1-t^2; the second-order term |f''|/2 dz^2 <= dz^2), plus the float32 evaluation of the gate
    functions and of c1 = sf*c0 + si*tj, h1 = so*tanh(c1) (ELEM, relative to the magnitudes involved).  A saturated gate
    is held to ~ELEM: its derivative, and with it its share of the z error, vanishes."""
    if dz is None:
        dz = zbar * float(np.max(np.abs(ref["z"])))
    g = ref["gates"]
    L = g.shape[1] // 4                 # the cell width (IMPALA 256, R2D2 64)
    si, tj, sf, so = g[:, :L], g[:, L:2 * L], g[:, 2 * L:3 * L], g[:, 3 * L:]
    deriv = np.concatenate([si * (1 - si), 1 - tj ** 2, sf * (1 - sf), so * (1 - so)], axis=1)
    eg = deriv * dz + dz ** 2 + ELEM
    ei, ej, ef, eo = eg[:, :L], eg[:, L:2 * L], eg[:, 2 * L:3 * L], eg[:, 3 * L:]
    ec = np.abs(c0) * ef + np.abs(tj) * ei + np.abs(si) * ej + ei * ej + ELEM * (np.abs(sf * c0) + np.abs(si * tj))
    tc = np.tanh(ref["c1"])
    eh = np.abs(tc) * eo + (so + eo) * ((1 - tc ** 2) * ec + ec ** 2) + ELEM
    return {"gates": eg, "c1": ec, "h1": eh}


def launch_facts(B, T):
    """Edges math mode 5 reaches at this shape: partial last M tiles of the 16-bit GEMMs (the M dimension of each launch
    of csrc/layers.cu over the tile the library reports), split-K counts of the conv weight gradients and frames per CTA
    of the persistent conv1 kernels -- the plan the library itself launches (drl_debug_launch_plan); more than two frames
    per CTA wraps the phase of the double-buffered frame barriers."""
    import ctypes
    from distributed_reinforcement_learning_b200 import _native as N
    out = (ctypes.c_int32 * 6)()
    N.check(N.lib.drl_debug_launch_plan(B, T, 5, out))
    M, Mb, tile = B * T, B * (T - 2), out[5]
    rows = {"lstm_fwd/heads_fwd": M, "heads_dgrad/lstm_dgrad": Mb, "conv2_fwd": M * 81, "conv3_fwd": M * 49,
            "conv3_dgrad": Mb * 81, "conv2_dgrad": Mb * 100}
    return dict(partial_tiles=sorted(k for k, r in rows.items() if r % tile),
                splits={"conv1_wgrad": out[0], "conv2_wgrad": out[1], "conv3_wgrad": out[2]},
                conv1_fwd_frames_per_cta=out[3], conv1_wgrad_frames_per_cta=out[4])


# ------------------------------------------------------------------------------------------------------------------
# regimes
# ------------------------------------------------------------------------------------------------------------------
REGIMES = ("init", "scaled", "trained", "conv1_w_1e-4", "conv1_w_5")
TRAIN_STEPS, TRAIN_LR = 20, 0.03
SCALE_LSTM, SHIFT_CONV3_B = 20.0, -0.05


def regime_params(regime, A):
    """The parameters a regime starts from (float32 values in a float64 OrderedDict); ``trained`` starts from init."""
    p = it.init_params(0, torch.float32, num_action=A)
    if regime == "scaled":
        # LSTM pre-activations ~20x (|z| > 4 for about a third of them: saturated gates), conv3 mostly dead
        p["lstm.w"] = p["lstm.w"] * SCALE_LSTM
        p["conv3.b"] = torch.full_like(p["conv3.b"], SHIFT_CONV3_B)
    elif regime.startswith("conv1_w_"):
        # conv1.w rescaled to a typical |w| of 1e-4 (the fp16 lo plane underflows into subnormals) or 5; conv2.w by
        # the inverse so that a2 and everything after it stay in the init range (biases are zero)
        target = float(regime[len("conv1_w_"):])
        s = target / float(p["conv1.w"].abs().median())
        p["conv1.w"] = (p["conv1.w"].double() * s).float()
        p["conv2.w"] = (p["conv2.w"].double() / s).float()
    return p


def run_case(mode, B, T, A, regime, seed=4242):
    """One step of a fresh learner in ``regime``; returns (rows, facts): rows = [dict(kernel, tensor, err, block, where,
    bar, ok)], facts = what the case reached (launch edges, regime statistics)."""
    from distributed_reinforcement_learning_b200.learner import NativeLearner
    params = regime_params(regime, A)
    cfg = dict(trajectory=T, num_action=A)
    eng = NativeLearner(batch=B, trajectory=T, num_action=A, math_mode=mode,
                        start_learning_rate=TRAIN_LR if regime == "trained" else it.DEFAULT_CFG["start_learning_rate"])
    facts = {}
    try:
        flat0 = it.flatten_params(params)
        eng.set_params(flat0)
        if regime == "trained":
            for s in range(TRAIN_STEPS):
                b = synthetic.make_batch(B, T=T, A=A, seed=10_000 + s)
                eng.stage(0, *[b[k] for k in synthetic.TRAIN_FIELDS])
                eng.step(0)
            flat = eng.get_params().astype(np.float64)
            facts["param_moved_rel_l2"] = float(np.linalg.norm(flat - flat0) / np.linalg.norm(flat0))
            trained = it.unflatten_params(flat, torch.float64, num_action=A)
            facts["biases_nonzero"] = all(bool(trained[k].abs().max() > 0) for k in trained if k.endswith(".b"))
        batch = synthetic.make_batch(B, T=T, A=A, seed=seed)
        buf, grads, p = run_step(eng, batch, B, T, A)
    finally:
        eng.close()
    ref = references(buf, p, batch, cfg, B, T, A)
    inp = device_inputs(batch)
    got = gpu_outputs(buf, grads, A)
    bar = bars(mode, B, T)
    per_element = dict(lstm_bounds(ref, inp["c0"], SPLIT16_LONGK if mode == 5 else TF32))
    if mode == 5:
        per_element["a1"] = conv1_bound(inp["x"], p["conv1.w"], p["conv1.b"])
    rows = []
    for name in KERNEL:
        if name in per_element:
            # per element against the bound of its error model (the relative errors are reported, the bound is the bar)
            ratio = float(np.max(np.abs(got[name] - ref[name]) / per_element[name]))
            e, blk, where = errors(name, got[name], ref[name])
            rows.append(dict(kernel=KERNEL[name], tensor=name, err=e, block=blk, where=where, bar="per-element bound",
                             bound_ratio=ratio, ok=bool(ratio <= 1.0)))
            continue
        e, blk, where = errors(name, got[name], ref[name])
        rows.append(dict(kernel=KERNEL[name], tensor=name, err=e, block=blk, where=where, bar=bar[name],
                         ok=bool(e <= bar[name] and blk <= bar[name])))
    facts["z_abs_gt4"] = float(np.mean(np.abs(ref["z"]) > 4))
    facts["a3_zero"] = float(np.mean(buf["a3"] <= 0))
    facts["conv1_w_median_abs"] = float(p["conv1.w"].abs().median())
    facts["finite"] = bool(all(np.all(np.isfinite(v)) for v in got.values()))
    return rows, facts
