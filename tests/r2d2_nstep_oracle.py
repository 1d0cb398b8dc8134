"""Float64 reference of the R2D2 learner's n-step double-Q targets and mixed max / mean sequence priorities (DESIGN.md
section 22), and the parity harness of the CUDA step in that mode.

``Learner`` is ``oracle/r2d2_torch.Learner`` with two more keyword arguments; with their defaults (n_step=1,
priority_eta=None) it computes exactly what its base class computes.  ``td_reference`` is the r2d2_td_nstep_kernel
check of ``tests/adam_layer_parity.r2d2_td`` (from the q values the step computed), with per-element bounds from the
float64 evaluation order: the return, the bootstrap and both rescalings in float64, rounded to float32 once."""
import numpy as np
import torch

from adam_layer_parity import U, _td_bounds
from apex_parity import adam_expected
from oracle import impala_torch as it
from oracle import r2d2_torch as rt
from parity import TOL, rel_err   # noqa: F401
from r2d2_parity import gpu_masks, r2d2_failures   # noqa: F401


def nstep_returns(target_q_boot, reward, done, bi, gamma, n):
    """G of every window i (t = bi + i) in float64, from the bootstrap values h^-1 is applied to:
    ``target_q_boot[b, i]`` = target_q[b, t + k][argmax main_q[b, t + k]], k = min(n, S - 1 - t).  -> (G, k)."""
    reward = np.asarray(reward, np.float32).astype(np.float64)
    done = np.asarray(done).astype(bool)
    B, S = reward.shape
    Nt = S - bi - 1
    G = np.zeros((B, Nt))
    k = np.minimum(n, S - 1 - (bi + np.arange(Nt)))
    boot = rt.vf_rescale_inv(torch.from_numpy(np.asarray(target_q_boot, np.float64))).numpy()
    for b in range(B):
        for i in range(Nt):
            t = bi + i
            ret, disc = 0.0, 1.0
            for j in range(k[i]):
                ret += disc * reward[b, t + j]
                disc *= 0.0 if done[b, t + j] else gamma
            G[b, i] = boot[b, i] * disc + ret
    return G, k


def bootstrap(main_q, target_q, bi, n, next_action=None):
    """target_q[b, t + k][a*] with a* = argmax main_q[b, t + k] (first maximum), or ``next_action[b, t + k - bi - 1]``
    when given (the argmax a step computed, over steps bi + 1 .. S - 1)."""
    mq, tq = np.asarray(main_q, np.float64), np.asarray(target_q, np.float64)
    B, S = mq.shape[:2]
    Nt = S - bi - 1
    u = bi + np.arange(Nt) + np.minimum(n, S - 1 - (bi + np.arange(Nt)))
    if next_action is None:
        arg = np.argmax(mq[:, u], axis=2)
    else:
        arg = np.asarray(next_action).astype(np.int64)[:, u - bi - 1]
    return np.take_along_axis(tq[:, u], arg[..., None], 2)[..., 0]


def priority(diff, eta):
    """Per-sequence priority of the windows' TD errors [B, Nt]: |mean diff| (eta None) or eta max |diff| + (1 - eta)
    mean |diff|, in float64."""
    diff = np.asarray(diff, np.float64)
    if eta is None:
        return np.abs(diff.mean(axis=1))
    a = np.abs(diff)
    return eta * a.max(axis=1) + (1.0 - eta) * a.mean(axis=1)


class Learner(rt.Learner):
    """oracle/r2d2_torch.Learner with the n-step target and the priority rule of DESIGN.md section 22."""

    def __init__(self, params=None, target_params=None, dtype=torch.float32, n_step=1, priority_eta=None, **cfg):
        super().__init__(params, target_params, dtype, **cfg)
        self.n_step, self.priority_eta = int(n_step), priority_eta

    def losses(self, state, previous_action, action, h, c, reward, done, weight=None, next_action=None):
        n = self.n_step
        if n <= 1:
            return super().losses(state, previous_action, action, h, c, reward, done, weight=weight,
                                  next_action=next_action)
        out = super().losses(state, previous_action, action, h, c, reward, done, weight=weight)
        bi = self.cfg["burn_in"]
        with torch.no_grad():
            boot = bootstrap(out["main_q"].numpy(), out["target_q"].numpy(), bi, n, next_action)
            G, _ = nstep_returns(boot, reward, done, bi, float(self.cfg["discount_factor"]), n)
            target = rt.vf_rescale(torch.from_numpy(G)).to(self.dtype)
        B = target.shape[0]
        w = (torch.ones(B, dtype=self.dtype) if weight is None
             else torch.from_numpy(np.asarray(weight, np.float32)).to(self.dtype))
        sav = out["state_action_value"]
        out["target_value"] = target
        out["value_loss"] = torch.mean(torch.mean((target - sav) ** 2, dim=1) * w)
        return out

    def get_td_error(self, state, previous_action, action, h, c, reward, done):
        with torch.no_grad():
            o = self.losses([state], [previous_action], [action], [h], [c], [reward], [done])
        return float(priority(o["target_value"].numpy() - o["state_action_value"].numpy(), self.priority_eta)[0])

    def train(self, state, previous_action, action, h, c, reward, done, weight, return_all=False, next_action=None):
        res, out, g, gn = super().train(state, previous_action, action, h, c, reward, done, weight, return_all=True,
                                        next_action=next_action)
        diff = out["target_value"].numpy() - out["state_action_value"].detach().numpy()
        res = (res[0], priority(diff, self.priority_eta))
        return (res, out, g, gn) if return_all else res


def td_reference(mq, tq, batch, bi, gamma, B, S, A, n_step=1, priority_eta=None):
    """adam_layer_parity.r2d2_td for the r2d2_td_nstep_kernel: the same references and ``bound/<name>`` entries from
    the q values the step computed ([B, S, A], batch-major), the target n-step and the priority by ``priority_eta``.
    The target is float64 throughout and rounded to float32 once, so its bound stays U |target|; the mixed priority
    adds the float32 rounding of its max, its warp-tree sum (depth <= 8) and its two products."""
    Nt = S - bi - 1
    t = bi + np.arange(Nt)
    mq, tq = np.asarray(mq, np.float64), np.asarray(tq, np.float64)
    boot = bootstrap(mq, tq, bi, n_step)
    G, _ = nstep_returns(boot, batch["reward"], batch["done"], bi, gamma, n_step)
    target = rt.vf_rescale(torch.from_numpy(G)).numpy()
    act = np.asarray(batch["action"]).astype(np.int64)[:, t]
    sav = np.take_along_axis(mq[:, t], act[..., None], 2)[..., 0]
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
    td = priority(diff, priority_eta)
    ref = dict(target_value=target, sav=sav, td=td, loss=float(np.mean(w[:, 0] * (diff ** 2).mean(1))), dq=dq,
               dmean=dmean)
    if priority_eta is None:
        ref["bound/td"] = ediff.mean(1) + 8 * U * np.abs(diff).mean(1) + U * td
    else:
        eta = priority_eta
        ref["bound/td"] = (eta * ediff.max(1) + (1 - eta) * (ediff.mean(1) + 10 * U * np.abs(diff).mean(1))
                           + 4 * U * td)
    ref["bound/loss"] = float(np.mean(w[:, 0] * (2 * np.abs(diff) * ediff + 16 * U * diff ** 2).mean(1)))
    ref["bound/target_value"] = U * np.abs(target)
    ref["bound/sav"] = np.zeros_like(sav)
    ref["bound/dq"], ref["bound/dmean"] = eq, em
    return ref


# ---- the CUDA step against the float64 oracle ------------------------------------------------------------------------

def make_batch(B, S, A, C, L, seed, done_rate=0.3):
    """rt.make_sequences at width L with dones redrawn at ``done_rate`` (dones fall inside the n-step horizons)."""
    b = rt.make_sequences(B, S=S, A=A, L=L, input_shape=(84, 84, C), seed=seed)
    if done_rate is not None:
        b["done"] = np.random.default_rng(seed + 7919).random((B, S)) < done_rate
    return b


def native(B, S, bi, A, C, L, params, target, **kw):
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET, NativeR2D2Learner
    eng = NativeR2D2Learner(batch=B, seq_len=S, burn_in=bi, num_action=A, lstm_size=L, input_shape=(84, 84, C), **kw)
    eng.set_params(rt.flatten_params(params), MAIN)
    eng.set_params(rt.flatten_params(target), TARGET)
    return eng


def compare_step(B, S, bi, n_step, priority_eta=None, A=4, C=1, L=64, seed=2468, steps=3, done_rate=0.3, **kw):
    """tests/r2d2_lstm_parity.compare_step in the n-step / mixed-priority mode: loss, taps, |td|, every gradient, the
    Adam update and slots against the float64 oracle over ``steps`` consecutive steps; ReLU kinks and double-Q argmax
    ties handled the same way (the oracle takes the step's own argmax at every bootstrap step)."""
    k = dict(num_action=A, lstm_size=L, input_shape=(84, 84, C))
    params = rt.init_params(0, torch.float32, **k)
    target = rt.init_params(1, torch.float32, **k)
    ref = Learner(params, target, torch.float64, n_step=n_step, priority_eta=priority_eta, seq_len=S, burn_in=bi, **k)
    eng = native(B, S, bi, A, C, L, params, target, n_step=n_step, priority_eta=priority_eta, **kw)
    errs = {}
    flips = elems = 0
    max_abs = 0.0
    disagree = 0
    try:
        for s in range(steps):
            tag = "" if steps == 1 else "@%d" % s
            b = make_batch(B, S, A, C, L, seed + s, done_rate)
            args = [b[x] for x in rt.TRAIN_FIELDS]
            st0 = eng.get_opt_state()
            p0 = eng.get_params()
            slot = s % eng.num_slots
            eng.stage(slot, b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"],
                      b["done"], b["weight"])
            out, td = eng.step(slot)
            taps = eng.taps()
            masks = gpu_masks(eng, B, S, A)
            with torch.no_grad():
                o0 = rt.Learner.losses(ref, *args[:-1], weight=args[-1])
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
            for x in ("main_q", "target_q", "target_value", "state_action_value"):
                errs["tap/" + x + tag] = rel_err(taps[x], o[x].detach().numpy())
            g_gpu = eng.get_grads()
            gd = rt.unflatten_params(g_gpu, torch.float64, **k)
            for x in grads:
                errs["grad/" + x + tag] = rel_err(gd[x].numpy(), grads[x].detach().numpy())
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
                for x in ref.params:
                    ref.params[x].copy_(pd[x])
                    ref.m[x].copy_(md[x])
                    ref.v[x].copy_(vd[x])
            ref.beta1_power, ref.beta2_power = np.float32(st1["beta1_power"]), np.float32(st1["beta2_power"])
        from distributed_reinforcement_learning_b200.r2d2_learner import TARGET
        tgt = rt.unflatten_params(eng.get_params(TARGET), torch.float64, **k)
        errs["target_unchanged"] = max(float((tgt[x] - ref.target[x]).abs().max()) for x in ref.target)
        errs["argmax/disagree_with_gap"] = float(disagree)
        errs["kink/flip_fraction"] = flips / max(elems, 1)
        errs["kink/max_abs_at_flip"] = max_abs
    finally:
        eng.close()
    return errs
