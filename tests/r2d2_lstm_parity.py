"""Parity harness of the R2D2 learner at lstm_size 256 and 512 (the cluster recurrence of csrc/r2d2_cluster.cuh): the
full step against the float64 oracle (``oracle/r2d2_torch.Learner(lstm_size=L)``) at the bar of tests/r2d2_parity.py,
and float64 references of the two recurrence kernels fed from the step's own buffers."""
import numpy as np
import torch

from apex_parity import adam_expected, check_opt
from oracle import impala_torch as it
from oracle import r2d2_torch as rt
from parity import TOL, rel_err   # noqa: F401
from r2d2_parity import gpu_masks, r2d2_failures   # noqa: F401

U32 = float(np.finfo(np.float32).eps) / 2


def kwp(A, L, C):
    return dict(num_action=A, lstm_size=L, input_shape=(84, 84, C))


def native(B, S, bi, A, C, L, params, target, **kw):
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET, NativeR2D2Learner
    eng = NativeR2D2Learner(batch=B, seq_len=S, burn_in=bi, num_action=A, lstm_size=L, input_shape=(84, 84, C), **kw)
    eng.set_params(rt.flatten_params(params), MAIN)
    eng.set_params(rt.flatten_params(target), TARGET)
    return eng


def make_batch(B, S, A, C, L, seed, done_ends=False):
    """rt.make_sequences at width L; with ``done_ends`` its dones are redrawn at rate 0.3 and forced at the first and the
    last step of every sequence (so a done falls at t = 0, mid-sequence and t = S - 1)."""
    b = rt.make_sequences(B, S=S, A=A, L=L, input_shape=(84, 84, C), seed=seed)
    if done_ends:
        b["done"] = np.random.default_rng(seed + 7919).random((B, S)) < 0.3
        b["done"][:, 0] = b["done"][:, S - 1] = True
    return b


def setup(B, S, bi, A, C, L, seed=0, opt=None, **kw):
    """(oracle Learner, CUDA learner) with the same initial parameters."""
    k = kwp(A, L, C)
    params = rt.init_params(seed, torch.float32, **k)
    target = rt.init_params(seed + 1, torch.float32, **k)
    ref = rt.Learner(params, target, torch.float64, seq_len=S, burn_in=bi, **k, **(opt or {}))
    return ref, native(B, S, bi, A, C, L, params, target, **(opt or {}), **kw)


def compare_step(B, S, bi, A=4, C=1, L=256, seed=2468, steps=1, done_ends=True, opt=None, **kw):
    """tests/r2d2_parity.compare_step at width L: taps, loss, |td|, every gradient, the Adam update and slots, against
    the float64 oracle; ReLU kinks and double-Q argmax ties handled the same way."""
    opt = check_opt(opt, ("learning_rate",))
    k = kwp(A, L, C)
    ref, eng = setup(B, S, bi, A, C, L, opt=opt, **kw)
    errs = {}
    flips = elems = 0
    max_abs = 0.0
    disagree = 0
    try:
        for s in range(steps):
            tag = "" if steps == 1 else "@%d" % s
            b = make_batch(B, S, A, C, L, seed + s, done_ends)
            args = [b[n] for n in rt.TRAIN_FIELDS]
            st0 = eng.get_opt_state()
            p0 = eng.get_params()
            slot = s % eng.num_slots
            eng.stage(slot, b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"],
                      b["done"], b["weight"])
            out, td = eng.step(slot)
            taps = eng.taps()
            masks = gpu_masks(eng, B, S, A)
            with torch.no_grad():
                o0 = ref.losses(*args[:-1], weight=args[-1])
            nq = o0["main_q"].numpy()[:, bi + 1:]
            gpu_na = np.argmax(taps["main_q"][:, bi + 1:], axis=2)
            top2 = np.sort(nq, axis=2)[..., -2:]
            disagree += int(np.sum((gpu_na != np.argmax(nq, axis=2)) & ((top2[..., 1] - top2[..., 0]) > 1e-5)))
            with it.activation_pattern(masks) as stt:
                res, o, grads, gn = ref.train(*args, return_all=True, next_action=gpu_na)
            flips, elems, max_abs = flips + stt["flips"], elems + stt["elems"], max(max_abs, stt["max_abs_at_flip"])
            errs["loss" + tag] = rel_err(out["loss"], res[0])
            errs["td_error" + tag] = rel_err(td, res[1])
            errs["grad_norm" + tag] = rel_err(out["grad_norm"], gn)
            if out["step"] != s + 1:
                errs["step" + tag] = float("inf")
            for n in ("main_q", "target_q", "target_value", "state_action_value"):
                errs["tap/" + n + tag] = rel_err(taps[n], o[n].detach().numpy())
            g_gpu = eng.get_grads()
            gd = rt.unflatten_params(g_gpu, torch.float64, **k)
            for n in grads:
                errs["grad/" + n + tag] = rel_err(gd[n].numpy(), grads[n].detach().numpy())
            st1 = eng.get_opt_state()
            p1 = eng.get_params()
            g64 = g_gpu.astype(np.float64)
            exp_p, exp_m, exp_v = adam_expected(p0.astype(np.float64), g64, st0["m"].astype(np.float64),
                                                st0["v"].astype(np.float64), float(np.sqrt(np.sum(g64 ** 2))), 1e30,
                                                float(np.float32(ref.cfg["learning_rate"])), st0["beta1_power"],
                                                st0["beta2_power"])
            floor = 4.0 * np.finfo(np.float32).eps * np.max(np.abs(p0)) / TOL
            errs["update/adam" + tag] = float(np.max(np.abs(p1 - exp_p)) / (np.max(np.abs(exp_p - p0)) + floor))
            errs["adam/m" + tag] = rel_err(st1["m"], exp_m)
            errs["adam/v" + tag] = rel_err(st1["v"], exp_v)
            pd = rt.unflatten_params(p1, torch.float64, **k)
            md = rt.unflatten_params(st1["m"], torch.float64, **k)
            vd = rt.unflatten_params(st1["v"], torch.float64, **k)
            with torch.no_grad():
                for n in ref.params:
                    ref.params[n].copy_(pd[n])
                    ref.m[n].copy_(md[n])
                    ref.v[n].copy_(vd[n])
            ref.beta1_power, ref.beta2_power = np.float32(st1["beta1_power"]), np.float32(st1["beta2_power"])
        from distributed_reinforcement_learning_b200.r2d2_learner import TARGET
        tgt = rt.unflatten_params(eng.get_params(TARGET), torch.float64, **k)
        errs["target_unchanged"] = max(float((tgt[n] - ref.target[n]).abs().max()) for n in ref.target)
        errs["argmax/disagree_with_gap"] = float(disagree)
        errs["kink/flip_fraction"] = flips / max(elems, 1)
        errs["kink/max_abs_at_flip"] = max_abs
    finally:
        eng.close()
    return errs


# ---- the recurrence kernels against float64, fed from the step's own buffers ----------------------------------------

def read_recurrence(eng, B, S, L):
    """The main scope's recurrence buffers of the last step, time-major [S, B, ...] float64."""
    M = B * S
    out = {}
    for n, w in (("zx", 4 * L), ("gates", 4 * L), ("tc", L), ("hout", L), ("hin", L), ("cin", L), ("dhout", L),
                 ("dz", 4 * L)):
        out[n] = eng.read_buffer(n, M * w).reshape(S, B, w).astype(np.float64)
    return out


def _split(z, L):
    return [z[..., k * L:(k + 1) * L] for k in range(4)]


def forward_check(buf, bias, Wh, done, L):
    """r2d2_lstm_fwd_cluster_kernel, step by step: z_t = zx + b + hin_t W_h from the kernel's own hin_t / cin_t, then
    gates, c_t, tanh(c_t), h_t.  Each element is held to a bound on float32 rounding: gamma_{L+8} (|zx| + |b| +
    sum |h||W|) on the pre-activation (FFMA chains over L terms plus the adds of <= 4 partial sums, in any order),
    8 u of the activation (expf / tanhf and the approximate division), and the first-order propagation through the
    cell.  The carried state must be hout / c masked by (1 - done), exactly for h.
    -> {name: worst |got - ref| / bound} (<= 1 passes)."""
    S = buf["zx"].shape[0]
    g = (L + 8) * U32 / (1 - (L + 8) * U32)
    pre = buf["zx"] + bias + buf["hin"] @ Wh
    mag = np.abs(buf["zx"]) + np.abs(bias) + np.abs(buf["hin"]) @ np.abs(Wh)
    e_pre = g * mag + 2 * U32 * np.abs(pre)
    i, j, f, o = _split(pre, L)
    si, tj, sf, so = 1 / (1 + np.exp(-i)), np.tanh(j), 1 / (1 + np.exp(-(f + 1))), 1 / (1 + np.exp(-o))
    gates = np.concatenate([si, tj, sf, so], -1)
    ei, ej, ef, eo = _split(e_pre, L)
    dg = np.concatenate([si * (1 - si) * ei, (1 - tj ** 2) * ej, sf * (1 - sf) * ef, so * (1 - so) * eo], -1)
    b_gates = dg + 8 * U32 * np.abs(gates) + 1e-30
    gi, gj, gf, go = _split(buf["gates"], L)         # the cell from the kernel's own gates
    c = gf * buf["cin"] + gi * gj
    b_c = 3 * U32 * (np.abs(gf * buf["cin"]) + np.abs(gi * gj)) + 1e-30
    tcv = np.tanh(c)
    b_tc = (1 - tcv ** 2) * b_c + 6 * U32 * np.abs(tcv) + 1e-30
    h = go * buf["tc"]
    b_h = 2 * U32 * np.abs(h) + 1e-30
    r = {"gates": np.max(np.abs(buf["gates"] - gates) / b_gates),
         "tc": np.max(np.abs(buf["tc"] - tcv) / b_tc),
         "hout": np.max(np.abs(buf["hout"] - h) / b_h)}
    keep = (1 - done.T.astype(np.float64))[..., None]          # [S, B, 1]
    r["hin_carry"] = 0.0 if np.array_equal(buf["hin"][1:], buf["hout"][:-1] * keep[:-1]) else np.inf
    r["cin_carry"] = np.max(np.abs(buf["cin"][1:] - c[:-1] * keep[:-1]) / b_c[:-1]) if S > 1 else 0.0
    return {k: float(v) for k, v in r.items()}


def backward_reference(buf, Wh, done, L):
    """BPTT of r2d2_lstm_bwd_cluster_kernel in float64 from the step's dhout, gates, tc, cin and done: dz [S, B, 4L]."""
    S, B = buf["dhout"].shape[:2]
    si, tj, sf, so = _split(buf["gates"], L)
    tcv, cin = buf["tc"], buf["cin"]
    keep = (1 - done.T.astype(np.float64))[..., None]
    dz = np.zeros((S, B, 4 * L))
    dh_in = np.zeros((B, L))
    dc_carry = np.zeros((B, L))
    for t in range(S - 1, -1, -1):
        dh = buf["dhout"][t] + keep[t] * dh_in
        d_o = dh * tcv[t] * so[t] * (1 - so[t])
        dc = keep[t] * dc_carry + dh * so[t] * (1 - tcv[t] ** 2)
        di = dc * tj[t] * si[t] * (1 - si[t])
        dj = dc * si[t] * (1 - tj[t] ** 2)
        df = dc * cin[t] * sf[t] * (1 - sf[t])
        dc_carry = dc * sf[t]
        dz[t] = np.concatenate([di, dj, df, d_o], -1)
        dh_in = dz[t] @ Wh.T
    return dz


def backward_error(buf, Wh, done, L):
    """Worst |dz - ref| over the largest |ref| of its i / j / f / o block, over the whole sequence."""
    ref = backward_reference(buf, Wh, done, L)
    return max(float(np.max(np.abs(a - r)) / max(np.max(np.abs(r)), 1e-30))
               for a, r in zip(_split(buf["dz"], L), _split(ref, L)))
