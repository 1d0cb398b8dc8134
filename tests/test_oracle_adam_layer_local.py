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
def test_r2d2_references_reproduce_oracle():
    """Dones in mid-sequence (the carry is cut inside the window and inside the burn-in) and burn-in > 0."""
    B, S, bi, A, C = 2, 6, 2, 3, 1
    kw = dict(num_action=A, lstm_size=64, input_shape=(84, 84, C))
    batch = r2d2_parity.make_batch(B, S, A, C, seed=31)
    batch["done"][:] = False
    batch["done"][0, 1] = batch["done"][1, 3] = True
    params = _params(rt.init_params(0, torch.float64, **kw))
    target = rt.init_params(1, torch.float64, **kw)
    L = rt.Learner(params, target, torch.float64, seq_len=S, burn_in=bi, **kw)
    o = L.losses(*[batch[k] for k in rt.TRAIN_FIELDS[:-1]], weight=batch["weight"])
    taps = o["taps"]
    acts = [taps[t][k] for t in range(S) for k, _ in CONV]
    grads, ag = _act_grads(o["value_loss"], L.params, acts)
    M = B * S
    buf = {}
    for ci, (k, shp) in enumerate(CONV):
        a = np.stack([_np(taps[t][k]) for t in range(S)]).reshape((M,) + shp)        # time-major
        d = np.stack([ag[t * len(CONV) + ci] for t in range(S)]).reshape((M,) + shp) * (a > 0)
        buf[k], buf["d" + k] = (a.reshape(M, -1), d.reshape(M, -1)) if k == "a3" else (a, d)
    mq, tq = _np(o["main_q"]), _np(o["target_q"])
    buf["q"] = lp.time_major(mq)
    shapes = {"e1": (A, 256), "emb": (A, 256), "zx": (M, 256), "gates": (M, 256), "tc": (M, 64), "hout": (M, 64),
              "q1": (M, 128), "dq1": (M, 128), "dhout": (M, 64), "dz": (M, 256), "du": (M, 256)}
    buf.update({k: np.zeros(s) for k, s in shapes.items()})
    inp = alp.r2d2_inputs(batch)
    keep = (~inp["done"]).astype(np.float64).T.reshape(M, 1)
    buf["hin"] = np.concatenate([inp["h0"], np.zeros((M - B, 64))])
    buf["cin"] = np.concatenate([inp["c0"], np.zeros((M - B, 64))])
    td = alp.r2d2_td(mq, tq, batch, bi, L.cfg["discount_factor"], B, S, A)
    buf["dq"], buf["dmean"] = np.zeros((M, 32)), np.zeros((M, 32))
    buf["dq"][:, :A], buf["dmean"][:, 0] = td["dq"], td["dmean"]
    state = {}

    def step(b):
        ref = alp.r2d2_references(b, L.params, batch, B, S, A)
        for k in shapes:
            b[k] = ref[k]
        b["hin"] = np.concatenate([inp["h0"], (ref["hout"] * keep)[:M - B]])
        b["cin"] = np.concatenate([inp["c0"], ref["cnext"]])
        state["ref"] = ref
    _converge(step, buf, 2 * S + 10)
    ref = state["ref"]
    errs = {}
    for k, _ in CONV:
        errs[k] = parity.rel_err(ref[k], buf[k])
    for k in ("da3", "da2", "da1"):
        errs[k] = parity.rel_err(ref[k], buf[k])
    errs["q"] = parity.rel_err(ref["q"], buf["q"])
    errs["gates"] = parity.rel_err(ref["gates"], alp._gates(ref["z"]))
    errs["tc"] = parity.rel_err(ref["tc"], np.tanh(ref["c"]))
    for k, ok in (("target_value", "target_value"), ("sav", "state_action_value")):
        errs[k] = parity.rel_err(td[k], _np(o[ok]))
    errs["loss"] = parity.rel_err(td["loss"], float(o["value_loss"].detach()))
    for n in grads:
        errs["grad/" + n] = parity.rel_err(ref[n], grads[n])
    assert len([k for k in errs if k.startswith("grad/")]) == 18
    assert all(np.abs(buf[k]).max() > 0 for k in shapes), "a derived buffer is all zero"
    # the window, the burn-in and the cut carry are all exercised
    assert np.abs(td["dq"]).max() > 0 and inp["done"][:, :S - 1].any() and bi > 0
    bad = _bad(errs)
    assert not bad, bad
