"""Parity harness of the R2D2 learner: the CUDA step (through ``drl_r2d2_*``) against the float64 CPU oracle
(``oracle/r2d2_torch.py``) on the same seeded sequences; same bar (1e-4 relative), ReLU-kink handling, double-Q argmax
handling and Adam check as tests/apex_parity.py."""
import numpy as np
import torch

from apex_parity import adam_expected, check_opt, load_adam_state
from oracle import impala_torch as it
from oracle import r2d2_torch as rt
from parity import TOL, failures, rel_err   # noqa: F401


def native_r2d2(B, S, bi, A, C, params, target, **kw):
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET, NativeR2D2Learner
    eng = NativeR2D2Learner(batch=B, seq_len=S, burn_in=bi, num_action=A, input_shape=(84, 84, C), **kw)
    eng.set_params(rt.flatten_params(params), MAIN)
    eng.set_params(rt.flatten_params(target), TARGET)
    return eng


def gpu_masks(eng, B, S, A):
    M = B * S

    def tm(name, per_row, shape):       # time-major device rows -> [S, B, ...]
        return torch.from_numpy(eng.read_buffer(name, M * per_row).reshape((S, B) + shape) > 0)
    return {"a1": tm("a1", 20 * 20 * 32, (20, 20, 32)), "a2": tm("a2", 9 * 9 * 64, (9, 9, 64)),
            "a3": tm("a3", 7 * 7 * 64, (7, 7, 64)), "q1": tm("q1", 128, (128,)),
            "e1": torch.from_numpy(eng.read_buffer("e1", A * 256).reshape(A, 256) > 0),
            "emb": torch.from_numpy(eng.read_buffer("emb", A * 256).reshape(A, 256) > 0)}


def make_batch(B, S, A, C, seed, done_rate=None, done_ends=False, L=64):
    """rt.make_sequences (h, c of width ``L``), optionally with its dones redrawn at ``done_rate`` and, with
    ``done_ends``, forced at the first and the last step of every sequence."""
    b = rt.make_sequences(B, S=S, A=A, L=L, input_shape=(84, 84, C), seed=seed)
    if done_rate is not None:
        b["done"] = np.random.default_rng(seed + 7919).random((B, S)) < done_rate
    if done_ends:
        b["done"][:, 0] = b["done"][:, S - 1] = True
    return b


def compare_step(B, S=15, bi=7, A=4, C=1, seed=2468, steps=1, sync_target_at=None, opt=None, init_state=None,
                 trace=None, done_rate=None, done_ends=False, **kw):
    """``opt``: dict(learning_rate=...) given to both the CUDA learner and the oracle (R2D2 does not clip);
    ``init_state`` and ``trace`` as in apex_parity.compare_step; ``done_rate`` / ``done_ends`` as in make_batch."""
    opt = check_opt(opt, ("learning_rate",))
    kwp = dict(num_action=A, lstm_size=64, input_shape=(84, 84, C))
    params = rt.init_params(0, torch.float32, **kwp)
    target = rt.init_params(1, torch.float32, **kwp)
    L = rt.Learner(params, target, torch.float64, seq_len=S, burn_in=bi, **kwp, **opt)
    eng = native_r2d2(B, S, bi, A, C, params, target, **opt, **kw)
    step0 = 0
    if init_state is not None:
        step0 = load_adam_state(eng, L, init_state, lambda f: rt.unflatten_params(f, torch.float64, **kwp))
    errs = {}
    flips = elems = 0
    max_abs = 0.0
    disagree = 0
    try:
        for s in range(steps):
            tag = "" if steps == 1 else "@%d" % s
            if sync_target_at is not None and s == sync_target_at:
                eng.main_to_target()
                L.main_to_target()
            b = make_batch(B, S, A, C, seed + s, done_rate, done_ends)
            args = [b[k] for k in rt.TRAIN_FIELDS]
            st0 = eng.get_opt_state()
            p0 = eng.get_params()
            slot = s % eng.num_slots
            eng.stage(slot, b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"],
                      b["done"], b["weight"])
            out, td = eng.step(slot)
            if trace is not None:
                trace.append(out)
            taps = eng.taps()
            masks = gpu_masks(eng, B, S, A)
            with torch.no_grad():
                o0 = L.losses(*args[:-1], weight=args[-1])
            nq = o0["main_q"].numpy()[:, bi + 1:]
            gpu_na = np.argmax(taps["main_q"][:, bi + 1:], axis=2)
            top2 = np.sort(nq, axis=2)[..., -2:]
            disagree += int(np.sum((gpu_na != np.argmax(nq, axis=2)) & ((top2[..., 1] - top2[..., 0]) > 1e-5)))
            with it.activation_pattern(masks) as stt:
                res, o, grads, gn = L.train(*args, return_all=True, next_action=gpu_na)
            flips, elems, max_abs = flips + stt["flips"], elems + stt["elems"], max(max_abs, stt["max_abs_at_flip"])
            errs["loss" + tag] = rel_err(out["loss"], res[0])
            errs["td_error" + tag] = rel_err(td, res[1])
            errs["grad_norm" + tag] = rel_err(out["grad_norm"], gn)
            if out["step"] != step0 + s + 1:
                errs["step" + tag] = float("inf")
            for k in ("main_q", "target_q", "target_value", "state_action_value"):
                errs["tap/" + k + tag] = rel_err(taps[k], o[k].detach().numpy())
            g_gpu = eng.get_grads()
            gd = rt.unflatten_params(g_gpu, torch.float64, **kwp)
            for n in grads:
                errs["grad/" + n + tag] = rel_err(gd[n].numpy(), grads[n].detach().numpy())
            if s == 0:      # forward activations of the main unroll, time-major
                for nm, shp in (("a1", (20, 20, 32)), ("a3", (7, 7, 64))):
                    got = eng.read_buffer(nm, B * S * int(np.prod(shp))).reshape((S, B) + shp)
                    ref = np.stack([o["taps"][t][nm].detach().numpy() for t in range(S)])
                    errs["act/" + nm] = rel_err(got, ref)
            st1 = eng.get_opt_state()
            p1 = eng.get_params()
            g64 = g_gpu.astype(np.float64)
            exp_p, exp_m, exp_v = adam_expected(p0.astype(np.float64), g64, st0["m"].astype(np.float64),
                                                st0["v"].astype(np.float64), float(np.sqrt(np.sum(g64 ** 2))), 1e30,
                                                float(np.float32(L.cfg["learning_rate"])), st0["beta1_power"],
                                                st0["beta2_power"])
            floor = 4.0 * np.finfo(np.float32).eps * np.max(np.abs(p0)) / TOL
            errs["update/adam" + tag] = float(np.max(np.abs(p1 - exp_p)) / (np.max(np.abs(exp_p - p0)) + floor))
            errs["adam/m" + tag] = rel_err(st1["m"], exp_m)
            errs["adam/v" + tag] = rel_err(st1["v"], exp_v)
            pd = rt.unflatten_params(p1, torch.float64, **kwp)
            md = rt.unflatten_params(st1["m"], torch.float64, **kwp)
            vd = rt.unflatten_params(st1["v"], torch.float64, **kwp)
            with torch.no_grad():
                for n in L.params:
                    L.params[n].copy_(pd[n])
                    L.m[n].copy_(md[n])
                    L.v[n].copy_(vd[n])
            L.beta1_power, L.beta2_power = np.float32(st1["beta1_power"]), np.float32(st1["beta2_power"])
        from distributed_reinforcement_learning_b200.r2d2_learner import TARGET
        tgt = rt.unflatten_params(eng.get_params(TARGET), torch.float64, **kwp)
        errs["target_unchanged"] = max(float((tgt[n] - L.target[n]).abs().max()) for n in L.target)
        errs["argmax/disagree_with_gap"] = float(disagree)
        errs["kink/flip_fraction"] = flips / max(elems, 1)
        errs["kink/max_abs_at_flip"] = max_abs
    finally:
        eng.close()
    return errs


def r2d2_failures(errs):
    bad = failures({k: v for k, v in errs.items() if not k.startswith(("target_unchanged", "argmax/"))})
    for k in ("target_unchanged", "argmax/disagree_with_gap"):
        if k in errs and not errs[k] == 0.0:
            bad[k] = errs[k]
    return bad
