"""Per-kernel float64 references of the policy engines' act, fed from the act's own buffers.

``policy_parity.compare_act``, ``r2d2_policy_parity`` and ``apex_policy_parity`` judge a whole act against the float64
oracle at 1e-4 of each output's maximum.  Here each kernel of the act is judged only from the buffers it read
(``PolicyHandle.read_buffer``: a1, a2, a3, e1, table, zpart) and the act's own outputs, with the oracle's layer
functions, as tests/layer_parity.py and tests/adam_layer_parity.py do for the learners.

Kernels of one act (csrc/policy.cu, r2d2_policy.cu, apex_policy.cu):
  * conv1 / conv2 / conv3: the learners' forwards at n <= 64 frames (IMPALA ``conv_forward16``, math mode 5, conv1 on
    fp16 split weights; R2D2, Ape-X and A3C ``conv_forward_tf32<C>``);
  * ``emb_forward``: e1 = relu(emb1) and the action-embedding table, from the parameters only;
  * ``skinny_splitk_fwd`` (policy_lstm.cuh): zpart[s] = x[:, Ks] W[Ks, :] over each split's own K range Ks, x =
    [a3 | table[pa] | h0] (IMPALA, R2D2) or [a3 | table[pa]] (Ape-X: W = [value1.w | mean1.w]; A3C: actor1.w).  Each
    element is one chain of kK fused multiply-adds from zero in K order, so |got - ref| <= gamma_kK sum_k |x_k w_k|
    (gamma_k = k u / (1 - k u), u = 2^-24) holds deterministically for the GPU's own float32 x and W;
  * the head: IMPALA ``policy_head_fused`` and R2D2 ``r2d2_policy_head`` sum the splits in index order, add the bias
    and form the LSTM cell (h', c' per element to ``layer_parity.lstm_bounds`` with the split sum's own per-element
    bound), then the actor head / q head from the act's h'; Ape-X / A3C ``apex_policy_head<algo>`` go from zpart + bias
    through the whole head (hid1, hid2 never leave shared memory);
  * the softmax (IMPALA, A3C) is also checked in log space, where the probabilities V-trace reads as log mu live;
  * the action rule, exactly, from the act's own q / policy.

Device conventions: zpart is [splits][n][N] with column c written by the CTA blockIdx.x = c // 128; the IMPALA, Ape-X
and A3C heads run 8 rows per CTA (blockIdx.x = row // 8), the R2D2 head one row per CTA.  A failure report names the
worst split, 128-column chunk and row (zpart) or the worst head CTA.
"""
import numpy as np
import torch

import adam_layer_parity as alp
import layer_parity as lp
from layer_parity import ELEM, FFMA_DOT, FLAT, SPLIT16, TF32, _np, _t
from oracle import a3c_torch as at
from oracle import apex_torch as ax
from oracle import impala_torch as it
from oracle import r2d2_torch as rt

U = 2.0 ** -24                  # float32 unit roundoff
U64 = 2.0 ** -53                # float64 unit roundoff (the references' own rounding)
EMB = 256
CHUNK = 128                     # columns per skinny CTA (policy_lstm.cuh kLN)
HEAD_ROWS = dict(impala=8, r2d2=1, apex=8, a3c=8)    # rows per head CTA
P_FLOOR = 1e-30                 # the log-space check covers every p_ref >= P_FLOOR
TINY = 1e-300

FAMILIES = ("impala", "r2d2", "apex", "a3c")
SPLITS = dict(impala=16, r2d2=48, apex=53, a3c=53)
COLS = dict(impala=1024, r2d2=256, apex=512, a3c=256)
TAIL = dict(impala=256, r2d2=64, apex=0, a3c=0)      # the h0 tail of x (the LSTM width); 0: no tail
ROWS = (1, 8, 9, 16, 17, 32, 33, 64)
MODULE = dict(impala=it, r2d2=rt, apex=ax, a3c=at)


def gamma(k, u=U):
    return k * u / (1 - k * u)


def row_tile(n):
    """The row tile R of the skinny GEMM instantiation launch_skinny_splitk picks for n rows (policy_lstm.cuh)."""
    for r in (8, 16, 32):
        if n <= r:
            return r
    return 64


def split_k(family):
    """Rows of W per split (kK)."""
    return (FLAT + EMB + TAIL[family]) // SPLITS[family]


def straddling_splits(family):
    """The splits whose K range crosses a part boundary of x ([a3 | table[pa] | h0]): the gather changes source
    inside them."""
    kK, K = split_k(family), FLAT + EMB + TAIL[family]
    return sorted({b // kK for b in (FLAT, FLAT + EMB) if b < K and b % kK})


# ------------------------------------------------------------------------------------------------------------------
# parameters and inputs
# ------------------------------------------------------------------------------------------------------------------
def _kw(family, A, C):
    kw = dict(num_action=A)
    if family == "r2d2":
        kw["input_shape"] = (84, 84, C)
    return kw


def init_params(family, A, C=1, seed=3):
    """The oracle's init_params with small nonzero biases (the initial biases are zero), float32 values."""
    p = MODULE[family].init_params(seed, torch.float32, **_kw(family, A, C))
    g = torch.Generator().manual_seed(seed + 1)
    for k in p:
        if k.endswith(".b"):
            p[k] = (torch.rand(p[k].shape, generator=g) - 0.5) * 0.2
    return p


def flatten(family, p):
    return (ax if family == "a3c" else MODULE[family]).flatten_params(p)


def unflatten(family, flat, A, C=1):
    return MODULE[family].unflatten_params(flat, torch.float64, **_kw(family, A, C))


def make_inputs(family, n, A, C=1, seed=7):
    """n rows of the family's act: state, pa (and h, c for the LSTM families), with the row selectors: ``u`` (IMPALA,
    A3C: one uniform draw per row) or ``explore`` (R2D2, Ape-X: -1 greedy on two rows of three, an action otherwise)."""
    import apex_policy_parity
    import policy_parity
    import r2d2_policy_parity
    if family == "impala":
        st, pa, h, c = policy_parity.make_inputs(n, A, seed)
        inp = dict(state=st, pa=pa, h=h, c=c)
    elif family == "r2d2":
        st, pa, h, c = r2d2_policy_parity.make_inputs(n, A, C, seed)
        inp = dict(state=st, pa=pa, h=h, c=c)
    else:
        st, pa = apex_policy_parity.make_inputs(n, A, seed)
        inp = dict(state=st, pa=pa)
    if family in ("impala", "a3c"):
        inp["u"] = np.random.RandomState(seed).random_sample(n)
    else:
        r = np.arange(n)
        inp["explore"] = np.where(r % 3 == 2, r % A, -1).astype(np.int32)
    return inp


def rows_of(inp, off, n):
    """Rows [off, off + n) of an input set."""
    return {k: np.ascontiguousarray(v[off:off + n]) for k, v in inp.items()}


# ------------------------------------------------------------------------------------------------------------------
# engines
# ------------------------------------------------------------------------------------------------------------------
def make_engine(family, A, C=1, max_batch=64):
    if family == "impala":
        from distributed_reinforcement_learning_b200.policy import NativePolicy
        return NativePolicy(max_batch, num_action=A)
    if family == "r2d2":
        from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
        return NativeR2D2Policy(max_batch, num_action=A, input_shape=(84, 84, C))
    from distributed_reinforcement_learning_b200.apex_policy import NativeA3CPolicy, NativeApexPolicy
    return (NativeApexPolicy if family == "apex" else NativeA3CPolicy)(max_batch, num_action=A)


def act(pol, family, inp):
    """One act of the engine on ``inp``; its outputs as float64 / int64 arrays."""
    if family == "impala":
        o = pol.act(inp["state"], inp["pa"], inp["h"], inp["c"], uniform=inp["u"])
        keys = ("action", "policy", "h", "c")
    elif family == "r2d2":
        o = pol.act(inp["state"], inp["pa"], inp["h"], inp["c"], explore_action=inp["explore"])
        keys = ("action", "q", "q_action", "h", "c")
    elif family == "apex":
        o = pol.act(inp["state"], inp["pa"], explore_action=inp["explore"])
        keys = ("action", "q", "q_action")
    else:
        o = pol.act(inp["state"], inp["pa"], uniform=inp["u"])
        keys = ("action", "policy", "max_prob")
    return {k: np.asarray(o[k], np.int64 if k == "action" else np.float64) for k in keys}


BUFFERS = ("a1", "a2", "a3", "e1", "table", "zpart")


def read_act(pol):
    """Every buffer of the engine's most recent act, float64, device layout."""
    return {k: pol.read_buffer(k).astype(np.float64) for k in BUFFERS}


# ------------------------------------------------------------------------------------------------------------------
# references
# ------------------------------------------------------------------------------------------------------------------
def first_weight(family, W):
    """The skinny GEMM's W [K, N]: lstm.w, [value1.w | mean1.w] (Ape-X) or actor1.w (A3C)."""
    if family in ("impala", "r2d2"):
        return W["lstm.w"]
    if family == "apex":
        return np.concatenate([W["value1.w"], W["mean1.w"]], axis=1)
    return W["actor1.w"]


def skinny_x(a3, table, pa, tail=None):
    """x = [a3 | table[pa] | tail] as the skinny GEMM gathers it."""
    parts = [np.asarray(a3, np.float64), np.asarray(table, np.float64)[np.asarray(pa, np.int64)]]
    if tail is not None:
        parts.append(np.asarray(tail, np.float64))
    return np.concatenate(parts, axis=1)


def skinny_references(x, W, splits):
    """(zpart reference [splits, n, N], per-element bound): each split over its own K range, bound gamma_kK sum |x w|
    (the float32 FFMA chain; plus the float64 reference's own rounding)."""
    n, K = x.shape
    kK = K // splits
    assert kK * splits == K and W.shape[0] == K
    ref = np.empty((splits, n, W.shape[1]))
    bound = np.empty_like(ref)
    ax_, aw = np.abs(x), np.abs(W)
    g = gamma(kK) + gamma(kK, U64)
    for s in range(splits):
        ks = slice(s * kK, (s + 1) * kK)
        ref[s] = x[:, ks] @ W[ks]
        bound[s] = g * (ax_[:, ks] @ aw[ks])
    return ref, bound


def gates_of(z):
    """[sigmoid(i) | tanh(j) | sigmoid(f + 1) | sigmoid(o)] (TF1 LSTMCell, forget bias 1)."""
    L = z.shape[1] // 4
    i, j, f, o = (z[:, k * L:(k + 1) * L] for k in range(4))
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))
    return np.concatenate([sig(i), np.tanh(j), sig(f + 1.0), sig(o)], axis=1)


def lstm_head_references(zpart, b, c0):
    """The LSTM cell of the IMPALA / R2D2 head from the GPU's zpart: z = sum_s zpart[s] + b, gates, c', h', and the
    per-element bounds of c' and h' (``layer_parity.lstm_bounds`` with dz = gamma_(S+1) (sum_s |zpart[s]| + |b|): the
    kernel adds the S partials in index order from zero, then the bias; the forget gate's + 1 is one more rounding)."""
    zpart = np.asarray(zpart, np.float64)
    S = zpart.shape[0]
    z = zpart.sum(0) + b
    g = gates_of(z)
    L = z.shape[1] // 4
    si, tj, sf, so = (g[:, k * L:(k + 1) * L] for k in range(4))
    c = sf * c0 + si * tj
    h = so * np.tanh(c)
    dz = gamma(S + 1) * (np.abs(zpart).sum(0) + np.abs(b))
    dz[:, 2 * L:3 * L] += U * np.abs(z[:, 2 * L:3 * L] + 1.0)
    bd = lp.lstm_bounds(dict(z=z, gates=g, c1=c), c0, None, dz=dz)
    return dict(z=z, gates=g, c=c, h=h, **{"bound/c": bd["c1"], "bound/h": bd["h1"]})


def _dense_relu(x, w, b):
    return np.maximum(x @ w + b, 0.0)


def log_softmax(logits):
    return _np(torch.log_softmax(_t(logits), dim=1))


def references(family, buf, out, P, inp, A):
    """{output: float64 reference} of one act, each from the GPU buffers its kernel read: the trunk from the frames
    and a1 / a2 (``layer_parity.trunk_forward_references``), zpart from a3 / table / h0, the head from zpart (Ape-X,
    A3C) or from zpart and the act's h' (IMPALA, R2D2).  ``P``: float64 parameters the act ran with; ``out``: the act's
    outputs.  Adds ``bound/<name>`` per-element bounds and ``logits`` (IMPALA, A3C)."""
    x = alp._frames(inp["state"])
    ref = lp.trunk_forward_references(buf, P, x, A, emb_key="table")
    W = {k: _np(v) for k, v in P.items()}
    if family == "impala":
        ref["bound/a1"] = lp.conv1_bound(x, P["conv1.w"], P["conv1.b"])
    xk = skinny_x(buf["a3"], buf["table"], inp["pa"], inp.get("h"))
    ref["zpart"], ref["bound/zpart"] = skinny_references(xk, first_weight(family, W), SPLITS[family])
    if family in ("impala", "r2d2"):
        ref.update(lstm_head_references(buf["zpart"], W["lstm.b"], np.asarray(inp["c"], np.float64)))
        h = out["h"]
        if family == "impala":
            hid = _dense_relu(_dense_relu(h, W["actor1.w"], W["actor1.b"]), W["actor2.w"], W["actor2.b"])
            ref["logits"] = hid @ W["actor3.w"] + W["actor3.b"]
            ref["policy"] = np.exp(log_softmax(ref["logits"]))
        else:
            q1 = _dense_relu(h, W["q1.w"], W["q1.b"])
            ref["q"] = (q1 @ W["value.w"] + W["value.b"]) - (q1 @ W["mean.w"] + W["mean.b"])
    else:
        streams = ("value", "mean") if family == "apex" else ("actor",)
        zsum = np.asarray(buf["zpart"], np.float64).sum(0)
        outs = []
        for z, s in enumerate(streams):
            hid1 = np.maximum(zsum[:, z * 256:(z + 1) * 256] + W[s + "1.b"], 0.0)
            hid2 = _dense_relu(hid1, W[s + "2.w"], W[s + "2.b"])
            outs.append(hid2 @ W[s + "3.w"] + W[s + "3.b"])
        if family == "apex":
            ref["q"] = outs[0] - outs[1]
        else:
            ref["logits"] = outs[0]
            ref["policy"] = np.exp(log_softmax(ref["logits"]))
    return ref


def expected_actions(family, out, inp):
    """The action rule applied to the act's own outputs: numpy's RandomState.choice for the row's draw (IMPALA, A3C),
    or the first maximum of q unless the row has an explore action (R2D2, Ape-X)."""
    import policy_parity
    if family in ("impala", "a3c"):
        n = out["policy"].shape[0]
        return np.array([policy_parity.expected_action(out["policy"][r], inp["u"][r]) for r in range(n)])
    greedy = np.argmax(out["q"], axis=1)
    return np.where(inp["explore"] >= 0, inp["explore"], greedy)


# ------------------------------------------------------------------------------------------------------------------
# metric
# ------------------------------------------------------------------------------------------------------------------
def _finite(x):
    return bool(np.all(np.isfinite(x)))


def _tensor_err(d, ref):
    mx = float(np.max(np.abs(ref))) if ref.size else 0.0
    return float(np.max(d)) / max(mx, 1e-30) if d.size else 0.0


def element_row(kernel, name, got, ref, bound, where_of):
    """A row held per element to ``bound``; ``where_of(index)`` names the worst element."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape == np.shape(bound), (name, got.shape, ref.shape, np.shape(bound))
    d = np.abs(got - ref)
    r = d / np.maximum(bound, TINY)
    if not _finite(got):
        r = np.where(np.isfinite(got), r, np.inf)
    i = np.unravel_index(int(np.argmax(r)), r.shape) if r.size else ()
    ratio = float(r[i]) if r.size else 0.0
    e = _tensor_err(d, ref)
    return dict(kernel=kernel, tensor=name, err=e, block=e, where=where_of(i) if r.size else "",
                bar="per-element bound", bound_ratio=ratio, ok=bool(ratio <= 1.0))


def splitk_row(kernel, got, ref, bound):
    """zpart per element to its FFMA-chain bound; the report names the worst split, 128-column chunk (the CTA's
    blockIdx.x) and row."""
    return element_row(kernel, "zpart", got, ref, bound,
                       lambda i: "split %d chunk %d row %d" % (i[0], i[2] // CHUNK, i[1]))


def pixel_row(kernel, name, got, ref, bar):
    """A conv activation per tensor and per 128-pixel block (rows of its [pixels, channels] view)."""
    C = np.shape(ref)[-1]
    g2, r2 = np.reshape(got, (-1, C)), np.reshape(ref, (-1, C))
    tiles = lambda nm, r: [("px%d" % s.start, s) for s in lp._row_tiles(r.shape[0])]
    e, blk, where = lp.errors(name, g2, r2, tiles)
    return dict(kernel=kernel, tensor=name, err=e, block=blk, where=where, bar=bar, ok=bool(e <= bar and blk <= bar))


def cta_blocks(rows_per_cta):
    """The head's CTA blocks: rows [k R, (k + 1) R) of a [n, A] output, labelled by blockIdx.x."""
    def f(name, ref):
        n, R = ref.shape[0], rows_per_cta
        return [("cta%d" % (r0 // R), slice(r0, min(r0 + R, n))) for r0 in range(0, n, R)]
    return f


def head_row(kernel, name, got, ref, rows_per_cta, bar=FFMA_DOT):
    e, blk, where = lp.errors(name, got, ref, cta_blocks(rows_per_cta))
    return dict(kernel=kernel, tensor=name, err=e, block=blk, where=where, bar=bar, ok=bool(e <= bar and blk <= bar))


def log_space_bound(logits_ref):
    """|log p - log p_ref| for p_ref >= P_FLOOR: a logit error of FFMA_DOT max|logit| moves log p by at most twice
    that (its own logit and the log of the sum), plus the float32 exp, sum and divide (8 u)."""
    return 2 * FFMA_DOT * float(np.max(np.abs(logits_ref))) + 8 * U


def log_space_row(kernel, got, logits_ref, rows_per_cta):
    """The softmax in log space: every p_ref >= P_FLOOR within ``log_space_bound`` (a probability the kernel flushed to
    zero, or normalised by another row's sum, fails)."""
    got = np.asarray(got, np.float64)
    lref = log_softmax(logits_ref)
    keep = np.exp(lref) >= P_FLOOR
    with np.errstate(divide="ignore", invalid="ignore"):
        d = np.where(keep, np.abs(np.log(got) - lref), 0.0)
    d = np.where(np.isnan(d), np.inf, d)
    b = log_space_bound(logits_ref)
    i = np.unravel_index(int(np.argmax(d)), d.shape)
    return dict(kernel=kernel, tensor="log policy", err=float(d[i]), block=float(d[i]),
                where="cta %d row %d action %d" % (i[0] // rows_per_cta, i[0], i[1]), bar="log-space bound",
                bound_ratio=float(d[i]) / b, ok=bool(d[i] <= b))


def exact_row(kernel, name, got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    bad = int(np.sum(got != ref))
    return dict(kernel=kernel, tensor=name, err=float(bad), block=float(bad), where="%d elements differ" % bad,
                bar="exact", ok=bad == 0)


HEAD_KERNEL = dict(impala="policy_head_fused", r2d2="r2d2_policy_head", apex="apex_policy_head<0>",
                   a3c="apex_policy_head<1>")
CONV_BAR = dict(impala=SPLIT16, r2d2=TF32, apex=TF32, a3c=TF32)


def check(family, buf, out, P, inp, A):
    """Rows (dict(kernel, tensor, err, block, where, bar, ok[, bound_ratio])) of every checked output of one act, and
    the references."""
    ref = references(family, buf, out, P, inp, A)
    hk, hr = HEAD_KERNEL[family], HEAD_ROWS[family]
    rows = []
    if family == "impala":
        rows.append(element_row("conv1_fwd", "a1", buf["a1"], ref["a1"], ref["bound/a1"],
                                lambda i: "frame %d px %d ch %d" % (i[0], i[1] * 20 + i[2], i[3])))
    else:
        rows.append(pixel_row("conv1_fwd", "a1", buf["a1"], ref["a1"], TF32))
    rows.append(pixel_row("conv2_fwd", "a2", buf["a2"], ref["a2"], CONV_BAR[family]))
    rows.append(pixel_row("conv3_fwd", "a3", buf["a3"].reshape(-1, 7, 7, 64), ref["a3"].reshape(-1, 7, 7, 64),
                          CONV_BAR[family]))
    rows.append(alp.bar_row("emb_forward", "e1", buf["e1"], ref["e1"], ELEM))
    rows.append(alp.bar_row("emb_forward", "table", buf["table"], ref["table"], FFMA_DOT))
    rows.append(splitk_row("skinny_splitk_fwd", buf["zpart"], ref["zpart"], ref["bound/zpart"]))
    if family in ("impala", "r2d2"):
        L = TAIL[family]
        for k in ("c", "h"):
            rows.append(element_row(hk, k, out[k], ref[k], ref["bound/" + k],
                                    lambda i: "cta %d row %d unit %d" % (i[0] // hr, i[0], i[1] % L)))
    if family in ("impala", "a3c"):
        rows.append(head_row(hk, "policy", out["policy"], ref["policy"], hr))
        rows.append(log_space_row(hk + "(softmax)", out["policy"], ref["logits"], hr))
    else:
        rows.append(head_row(hk, "q", out["q"], ref["q"], hr))
    rows.append(exact_row(hk + "(action)", "action", out["action"], expected_actions(family, out, inp)))
    n = out["action"].shape[0]
    sel = "max_prob" if family == "a3c" else "q_action"
    if sel in out:
        src = out["policy"] if family == "a3c" else out["q"]
        rows.append(exact_row(hk + "(action)", sel, out[sel], src[np.arange(n), out["action"]]))
    return rows, ref


# ------------------------------------------------------------------------------------------------------------------
# one act on the GPU
# ------------------------------------------------------------------------------------------------------------------
REGIMES = dict(impala=("init", "trained", "saturated", "peaked", "conv1_w_1e-4", "conv1_w_5"),
               r2d2=("init", "trained", "saturated"), apex=("init", "trained"), a3c=("init", "trained", "peaked"))
SCALE_LSTM = dict(impala=lp.SCALE_LSTM, r2d2=alp.SCALE_LSTM)     # saturated: >= 20 % of |z| > 4
PEAK_LOGIT = alp.PEAK_LOGIT                                       # peaked: logits spread over 45, min p ~ 3e-20


def regime_params(family, A, C, regime):
    """The parameters an act in ``regime`` starts from (``trained`` starts from init and trains a learner)."""
    if regime.startswith("conv1_w_"):
        return lp.regime_params(regime, A)
    p = init_params(family, A, C)
    if regime == "saturated":
        p["lstm.w"] = p["lstm.w"] * SCALE_LSTM[family]
    elif regime == "peaked":
        p["actor3.b"] = torch.linspace(0.0, -PEAK_LOGIT, A, dtype=torch.float32)
    return p


def train_and_sync(pol, family, A, C, params):
    """Trains a fresh learner of the family from ``params`` at a raised learning rate (layer_parity /
    adam_layer_parity's training settings) and syncs the engine from it; returns the regime facts."""
    from oracle import synthetic
    kw = _kw(family, A, C)
    flat0 = flatten(family, params)
    if family == "impala":
        from distributed_reinforcement_learning_b200.learner import NativeLearner
        B, T = 32, 20
        eng = NativeLearner(batch=B, trajectory=T, num_action=A, math_mode=5, start_learning_rate=lp.TRAIN_LR)
        eng.set_params(flat0)

        def stage(s):
            b = synthetic.make_batch(B, T=T, A=A, seed=s)
            eng.stage(0, *[b[k] for k in synthetic.TRAIN_FIELDS])
        steps = lp.TRAIN_STEPS
    elif family == "r2d2":
        import r2d2_parity
        from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET, NativeR2D2Learner
        B, S = 16, 15
        eng = NativeR2D2Learner(batch=B, seq_len=S, burn_in=7, num_action=A, input_shape=(84, 84, C), math_mode=2,
                                learning_rate=alp.TRAIN_LR)
        eng.set_params(flat0, MAIN)
        eng.set_params(rt.flatten_params(rt.init_params(1, torch.float32, **kw)), TARGET)

        def stage(s):
            b = r2d2_parity.make_batch(B, S, A, C, s, None, False)
            eng.stage(0, b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"],
                      b["done"], b["weight"])
        steps = alp.TRAIN_STEPS
    else:
        B = 32
        if family == "apex":
            from distributed_reinforcement_learning_b200.apex_learner import MAIN, TARGET, NativeApexLearner
            eng = NativeApexLearner(batch=B, num_action=A, math_mode=2, start_learning_rate=alp.TRAIN_LR)
            eng.set_params(flat0, MAIN)
            eng.set_params(ax.flatten_params(ax.init_params(1, torch.float32, **kw)), TARGET)
        else:
            from distributed_reinforcement_learning_b200.a3c_learner import NativeA3CLearner
            eng = NativeA3CLearner(batch=B, num_action=A, math_mode=2, start_learning_rate=alp.TRAIN_LR)
            eng.set_params(flat0)
        fields = ax.TRAIN_FIELDS if family == "apex" else at.TRAIN_FIELDS

        def stage(s):
            b = ax.make_transitions(B, A=A, seed=s)
            eng.stage(0, *[b[k] for k in fields])
        steps = alp.TRAIN_STEPS
    try:
        alp._train(eng, stage, steps)
        pol.sync_from(eng)
        flat = pol.get_params()          # waits for the engine's stream: the sync's copy is complete
    finally:
        eng.close()
    return alp._moved(flat0.astype(np.float64), flat, lambda f: unflatten(family, f, A, C))


def run_case(family, n, A, C=1, regime="init", pol=None, seed=7):
    """One act of n rows in ``regime`` on ``pol`` (a fresh engine when None); returns (rows, facts): rows as
    ``check``, facts = what the case reached (row tile, partial head CTA, regime statistics)."""
    own = pol is None
    if own:
        pol = make_engine(family, A, C)
    facts = dict(row_tile=row_tile(n), partial_head_cta=bool(n % HEAD_ROWS[family]))
    try:
        params = regime_params(family, A, C, regime)
        pol.set_params(flatten(family, params))
        if regime == "trained":
            facts.update(train_and_sync(pol, family, A, C, params))
        P = unflatten(family, pol.get_params(), A, C)
        inp = make_inputs(family, n, A, C, seed)
        out = act(pol, family, inp)
        buf = read_act(pol)
        facts["buffer_dims"] = pol.buffer_dims()
    finally:
        if own:
            pol.close()
    rows, ref = check(family, buf, out, P, inp, A)
    facts["finite"] = bool(all(_finite(v) for v in list(buf.values()) + list(out.values())))
    if "z" in ref:
        facts["z_abs_gt4"] = float(np.mean(np.abs(ref["z"]) > 4))
    if "logits" in ref:
        facts["policy_ref_min"] = float(np.exp(log_softmax(ref["logits"])).min())
    facts["conv1_w_median_abs"] = float(P["conv1.w"].abs().median())
    return rows, facts


def row_independence(pol, family, A, C=1, seed=11):
    """One 64-row act, then acts on the prefixes n = 33, 17, 9, 1 and on the window of rows [23, 40): for each of
    these and each buffer / output, the number of elements of its rows that differ from the same rows of the 64-row
    act (bitwise; zpart row by row in every split)."""
    inp = make_inputs(family, 64, A, C, seed)
    pol.set_params(flatten(family, init_params(family, A, C)))
    full = act(pol, family, inp)
    full.update(read_act(pol))
    diffs = {}
    for off, m in ((0, 33), (0, 17), (0, 9), (0, 1), (23, 17)):
        part = act(pol, family, rows_of(inp, off, m))
        part.update(read_act(pol))
        for k, v in part.items():
            if k in ("e1", "table"):
                w = full[k]
            elif k == "zpart":
                w = full[k][:, off:off + m]
            else:
                w = full[k][off:off + m]
            diffs["rows %d..%d/%s" % (off, off + m - 1, k)] = int(np.sum(v != w))
    return diffs
