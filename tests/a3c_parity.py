"""Parity harness of the A3C learner: the CUDA step (through ``drl_a3c_*``) against the float64 CPU oracle
(``oracle/a3c_torch.py``) on the same seeded minibatch; same bar (1e-4 relative), ReLU-kink handling and Adam check as
tests/apex_parity.py."""
import numpy as np
import torch

import apex_parity as ap
from oracle import a3c_torch as at
from oracle import impala_torch as it
from parity import TOL, rel_err


def masks(eng, B, A):
    m = ap.gpu_masks(eng, B, A)
    return {k.replace("value", "actor").replace("mean", "critic"): v for k, v in m.items()}


def native_a3c(B, A, params, **kw):
    from distributed_reinforcement_learning_b200.a3c_learner import NativeA3CLearner
    eng = NativeA3CLearner(batch=B, num_action=A, **kw)
    eng.set_params(at.flatten_params(params))
    return eng


def compare_step(B, A=4, seed=4321, steps=1, reward_clipping="abs_one", opt=None, init_state=None, trace=None, **kw):
    """``opt``, ``init_state`` and ``trace`` as in apex_parity.compare_step."""
    opt = ap.check_opt(opt)
    params = at.init_params(0, torch.float32, num_action=A)
    L = at.Learner(params, torch.float64, num_action=A, reward_clipping=reward_clipping, **opt)
    eng = native_a3c(B, A, params, reward_clipping=reward_clipping, **opt, **kw)
    step0 = 0
    if init_state is not None:
        step0 = ap.load_adam_state(eng, L, init_state, lambda f: at.unflatten_params(f, torch.float64, num_action=A))
    errs = {}
    flips = elems = 0
    max_abs = 0.0
    try:
        for s in range(steps):
            tag = "" if steps == 1 else "@%d" % s
            b = at.make_transitions(B, A=A, seed=seed + s)
            args = [b[k] for k in at.TRAIN_FIELDS]
            st0, p0 = eng.get_opt_state(), eng.get_params()
            eng.stage(s % eng.num_slots, *args)
            out = eng.step(s % eng.num_slots)
            if trace is not None:
                trace.append(out)
            taps = eng.taps()
            with it.activation_pattern(masks(eng, B, A)) as stt:
                res, o, grads, gn = L.train(*args, return_all=True)
            flips, elems, max_abs = flips + stt["flips"], elems + stt["elems"], max(max_abs, stt["max_abs_at_flip"])
            for i, k in enumerate(("pi_loss", "baseline_loss", "entropy")):
                errs["loss/" + k + tag] = rel_err(out[k], res[i])
            errs["lr" + tag] = abs(out["learning_rate"] - res[3])
            errs["grad_norm" + tag] = rel_err(out["grad_norm"], gn)
            if out["step"] != step0 + s + 1:
                errs["step" + tag] = float("inf")
            for k in ("policy", "value", "next_value", "advantage"):
                errs["tap/" + k + tag] = rel_err(taps[k], o[k].detach().numpy())
            g_gpu = eng.get_grads()
            gd = at.unflatten_params(g_gpu, torch.float64, num_action=A)
            for n in grads:
                errs["grad/" + n + tag] = rel_err(gd[n].numpy(), grads[n].detach().numpy())
            st1, p1 = eng.get_opt_state(), eng.get_params()
            g64 = g_gpu.astype(np.float64)
            exp_p, exp_m, exp_v = ap.adam_expected(p0.astype(np.float64), g64, st0["m"].astype(np.float64),
                                                   st0["v"].astype(np.float64), float(np.sqrt(np.sum(g64 ** 2))),
                                                   L.cfg["gradient_clip_norm"], float(out["learning_rate"]),
                                                   st0["beta1_power"], st0["beta2_power"])
            floor = 4.0 * np.finfo(np.float32).eps * np.max(np.abs(p0)) / TOL
            errs["update/adam" + tag] = float(np.max(np.abs(p1 - exp_p)) / (np.max(np.abs(exp_p - p0)) + floor))
            errs["adam/m" + tag] = rel_err(st1["m"], exp_m)
            errs["adam/v" + tag] = rel_err(st1["v"], exp_v)
            pd = at.unflatten_params(p1, torch.float64, num_action=A)
            md = at.unflatten_params(st1["m"], torch.float64, num_action=A)
            vd = at.unflatten_params(st1["v"], torch.float64, num_action=A)
            with torch.no_grad():
                for n in L.params:
                    L.params[n].copy_(pd[n])
                    L.m[n].copy_(md[n])
                    L.v[n].copy_(vd[n])
            L.beta1_power, L.beta2_power = np.float32(st1["beta1_power"]), np.float32(st1["beta2_power"])
        errs["kink/flip_fraction"] = flips / max(elems, 1)
        errs["kink/max_abs_at_flip"] = max_abs
    finally:
        eng.close()
    return errs
