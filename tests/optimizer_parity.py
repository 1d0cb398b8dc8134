"""Float64 references of the last part of every training step -- the global norm, the clip scale, the learning rate,
the Adam scalars and the per-element RMSProp / Adam update -- built from the float32 inputs the kernels read
(``sqnorm_partial_kernel`` / ``rmsprop_apply_kernel`` in csrc/optimizer.cu, ``adam_prepare_kernel`` /
``adam_apply_kernel`` in csrc/adam_learner.cu), with per-element error bounds derived from the float32 rounding of each
operation.

Rounding model (u = 2^-24, one rounding of a float32 result r adds at most u|r| + 2^-150, the second term being half
the smallest subnormal: the build does not flush denormals):

* every constant is the float32 value TF uses: 0.99f, 1 - 0.99f (exact), 0.1f, 0.9f, 0.999f, 1 - 0.9f, 1 - 0.999f,
  1e-8f;
* the library builds with nvcc's default ``--fmad=true`` and no fast math, so ``a * b + c`` may be one FMA or a product
  and a sum: the bounds allow the rounding of both, divisions and ``sqrtf`` are correctly rounded;
* ``rsqrtf`` is ``rsqrt.approx.f32``: at most 2 ulp (CUDA programming guide; the PTX ISA states a relative error of
  2^-22.9), taken here as a relative 2^-22;
* the global norm is reduced in float32 by a fixed tree: per-thread FMA chains over the float4 elements of a
  528 x 256 grid (4 * ceil(n / 4 / 135168) terms), a 5-level warp tree, an 8-way block sum, then in the apply kernel
  every block re-reduces the 528 partials (up to 3 per thread, a warp tree, 8 warps).  With d the depth of that tree
  the float32 sum of squares is within gamma_d * s of the exact s (gamma_d = d u / (1 - d u)).

The scalars are exact: the learning rate is ``impala_torch.polynomial_decay_f32`` bit for bit, ``alpha`` and the beta
powers are evaluated in float32 as ApplyAdam does, and the clip scale is computed in float32 from the norm the kernel
REPORTED (so each kernel is judged on its own inputs).  A NaN or infinite norm makes the scale NaN, as
``tf.clip_by_global_norm`` does (TF 1.14 clip_ops: ``scale_for_finite + (norm - norm)``)."""
import math

import numpy as np

from oracle import impala_torch as it

f32 = np.float32
U = 2.0 ** -24
ETA = 2.0 ** -150
RSQRT_REL = 2.0 ** -22
FLT_MAX = float(np.finfo(np.float32).max)
NBLK, THREADS = 132 * 4, 256          # the optimizer kernels' grid (learner.cu, adam_learner.cu)

RMS_DECAY, RMS_EPS = f32(0.99), f32(0.1)
RMS_C = f32(1) - RMS_DECAY            # 1 - 0.99f, exact in float32
BETA1, BETA2, ADAM_EPS = f32(0.9), f32(0.999), f32(1e-8)
ADAM_C1, ADAM_C2 = f32(1) - BETA1, f32(1) - BETA2


# ---- scalars --------------------------------------------------------------------------------------------------------
def learning_rate(start, end, learning_frame, step):
    """tf.train.polynomial_decay in float32 at the pre-increment step."""
    return f32(it.polynomial_decay_f32(start, step, learning_frame, end))


def adam_scalars(lr, b1p, b2p):
    """(alpha, beta1_power', beta2_power') of ApplyAdam in float32: alpha from the powers BEFORE they advance."""
    lr, b1p, b2p = f32(lr), f32(b1p), f32(b2p)
    alpha = f32(f32(lr * np.sqrt(f32(1) - b2p)) / (f32(1) - b1p))
    return alpha, f32(b1p * BETA1), f32(b2p * BETA2)


def clip_scale(norm, clip, grad_scale=1.0):
    """The factor the apply kernels multiply every gradient by, in float32, from the reported norm (which already
    includes ``grad_scale`` for the Adam families).  clip <= 0: no clipping (R2D2's ``minimize``)."""
    n = f32(norm)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if clip > 0:
            c = f32(clip)
            s = f32(c * np.minimum(f32(1) / n, f32(1) / c))
            s = f32(s + (n - n))
        else:
            s = f32(1)
        return f32(s * f32(grad_scale))


# ---- the global norm ------------------------------------------------------------------------------------------------
def norm_depth(padded_total, nblk=NBLK, threads=THREADS):
    """Roundings on the longest path of the float32 sum-of-squares tree."""
    chain = 4 * -(-(padded_total // 4) // (nblk * threads))
    return chain + 5 + 7 + -(-nblk // threads) + 5 + 7


def global_norm(g, padded_total, grad_scale=1.0):
    """-> (kind, norm, bound): the float64 norm of the packed gradient ``g`` times ``grad_scale`` and the bound on the
    float32 tree's error.  kind: "finite", "inf" (the float32 sum of squares overflows, or an element is infinite) or
    "nan".  An input whose float32 sum could land on either side of FLT_MAX is refused."""
    g64 = np.asarray(g, np.float32).astype(np.float64)
    if np.isnan(g64).any():
        return "nan", float("nan"), 0.0
    if np.isinf(g64).any():
        return "inf", float("inf"), 0.0
    s = float(np.dot(g64, g64))
    d = norm_depth(padded_total)
    gam = d * U / (1 - d * U)
    if s * (1 - gam) > FLT_MAX * (1 + U):
        return "inf", float("inf"), 0.0
    if s * (1 + gam) >= FLT_MAX:
        raise ValueError("sum of squares %.6g is within rounding of FLT_MAX" % s)
    err_s = gam * s + 2 * padded_total * ETA
    n = math.sqrt(s)
    err_n = min(err_s / (2 * n) if n > 0 else float("inf"), math.sqrt(err_s)) + U * (n + err_s) + ETA
    return "finite", n * grad_scale, err_n * grad_scale + ETA


def norm_ratio(got, g, padded_total, grad_scale=1.0):
    """|got - ref| / bound for a finite norm; 0 if a non-finite norm has the expected kind, else inf."""
    kind, ref, bound = global_norm(g, padded_total, grad_scale)
    got = float(got)
    if kind == "nan":
        return 0.0 if math.isnan(got) else float("inf")
    if kind == "inf":
        return 0.0 if got == float("inf") else float("inf")
    if not math.isfinite(got):
        return float("inf")
    return abs(got - ref) / bound


# ---- the per-element update -----------------------------------------------------------------------------------------
def _f64(*a):
    return [np.asarray(x, np.float32).astype(np.float64) for x in a]


def rmsprop(w, ms, g, scale, lr):
    """TF1 RMSProp (decay 0.99, epsilon 0.1 inside the square root, momentum 0) of the clipped gradient
    ``g * scale`` -> (dict(w, ms) in float64, dict of per-element bounds)."""
    w, ms, g = _f64(w, ms, g)
    s, lr, c, eps = float(f32(scale)), float(f32(lr)), float(RMS_C), float(RMS_EPS)
    with np.errstate(all="ignore"):
        gg = g * s
        e_gg = U * np.abs(gg) + ETA
        t = gg * gg - ms
        e_t = 2 * np.abs(gg) * e_gg + U * gg * gg + U * np.abs(t) + ETA
        m1 = ms + t * c
        e_m1 = c * e_t + U * np.abs(t * c) + U * np.abs(m1) + 2 * ETA
        a = m1 + eps
        e_a = e_m1 + U * np.abs(a) + ETA
        r = 1.0 / np.sqrt(a)
        e_r = 0.5 * r / (a - e_a) * e_a + RSQRT_REL * r
        p = lr * gg
        e_p = lr * e_gg + U * np.abs(p) + ETA
        q = p * r
        w1 = w - q
        e_w = r * e_p + np.abs(p) * e_r + U * np.abs(q) + U * np.abs(w1) + 2 * ETA
    return dict(w=w1, ms=m1), dict(w=e_w * (1 + 1e-6), ms=e_m1 * (1 + 1e-6))


def adam(w, m, v, g, scale, alpha):
    """TF1 ApplyAdam of the clipped gradient ``g * scale`` with the float32 ``alpha`` -> (dict(w, m, v) in float64,
    dict of per-element bounds)."""
    w, m, v, g = _f64(w, m, v, g)
    s, al, c1, c2, eps = (float(f32(scale)), float(f32(alpha)), float(ADAM_C1), float(ADAM_C2), float(ADAM_EPS))
    with np.errstate(all="ignore"):
        gg = g * s
        e_gg = U * np.abs(gg) + ETA
        d1 = gg - m
        e_d1 = e_gg + U * np.abs(d1) + ETA
        m1 = m + d1 * c1
        e_m1 = c1 * e_d1 + U * np.abs(d1 * c1) + U * np.abs(m1) + 2 * ETA
        t = gg * gg - v
        e_t = 2 * np.abs(gg) * e_gg + U * gg * gg + U * np.abs(t) + ETA
        v1 = v + t * c2
        e_v1 = c2 * e_t + U * np.abs(t * c2) + U * np.abs(v1) + 2 * ETA
        sq = np.sqrt(v1)
        e_sq = np.minimum(np.where(sq > 0, e_v1 / (2 * sq), np.inf), np.sqrt(e_v1)) + U * sq + ETA
        den = sq + eps
        e_den = e_sq + U * den
        num = m1 * al
        e_num = al * e_m1 + U * np.abs(num) + ETA
        q = num / den
        e_q = (e_num + np.abs(q) * e_den) / (den - e_den) + U * np.abs(q) + ETA
        w1 = w - q
        e_w = e_q + U * np.abs(w1) + ETA
    k = 1 + 1e-6
    return dict(w=w1, m=m1, v=v1), dict(w=e_w * k, m=e_m1 * k, v=e_v1 * k)


def ratio(got, ref, bound):
    """-> (worst |got - ref| / bound, its index).  Where the reference is not finite the kernel must produce the same
    value (NaN for NaN); a finite reference needs a finite result."""
    got = np.asarray(got, np.float32).astype(np.float64)
    ref = np.asarray(ref, np.float64)
    fin = np.isfinite(ref)
    same = (np.isnan(ref) & np.isnan(got)) | (ref == got)
    bad = (~fin & ~same) | (fin & ~np.isfinite(got))
    if bad.any():
        return float("inf"), int(np.flatnonzero(bad)[0])
    if not fin.any():
        return 0.0, -1
    with np.errstate(all="ignore"):
        r = np.where(fin, np.abs(got - ref) / bound, 0.0)
    i = int(np.argmax(r))
    return float(r[i]), i


# ---- the gradient bucket -------------------------------------------------------------------------------------------
def bucket_index_map(eng):
    """-> (packed_to_padded int64 [param_count], padded_total) of a learner handle: writes bucket[i] = i through the
    bucket view and reads it back with ``get_grads`` (padded_total < 2^24, so every index is exact in float32).  The
    padding elements are the indices that do not appear.  The bucket is restored afterwards (the backward pass never
    writes its padding, so it keeps whatever is there)."""
    import torch
    b = eng._dp._tensor()
    npad = b.numel() - 4
    assert npad < 2 ** 24
    with torch.cuda.stream(eng._dp._stream):
        saved = b.clone()
        b[:npad] = torch.arange(npad, dtype=torch.float32, device=b.device)
    eng._dp._stream.synchronize()
    idx = eng.get_grads().astype(np.int64)
    with torch.cuda.stream(eng._dp._stream):
        b.copy_(saved)
    eng._dp._stream.synchronize()
    assert len(np.unique(idx)) == idx.size and idx.min() >= 0 and idx.max() < npad
    return idx, npad


def padding_of(idx, npad):
    mask = np.ones(npad, bool)
    mask[idx] = False
    return np.flatnonzero(mask)
