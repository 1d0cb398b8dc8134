"""Float64 oracle of the IMPALA learner's recurrent mode (``NativeLearner(..., recurrent=True)``, DESIGN.md section 21)
and its GPU parity harness -- TEST INFRASTRUCTURE ONLY.

``RecurrentLearner`` is ``oracle.impala_torch.Learner`` with the LSTM run through the T steps of each trajectory:
  h_in(0), c_in(0) = the recorded initial_h[:, 0], initial_c[:, 0]
  h_in(t), c_in(t) = initial_h[:, t], initial_c[:, t] if done[:, t-1] else h_out(t-1), c_out(t-1)    (t >= 1)
and autograd through the unroll (so no gradient crosses a done, and the recorded states receive none).  Everything
downstream (heads, V-trace windows, losses, clip, RMSProp) is the parent class's.

``bug`` injects one known defect of a GPU implementation, for the tests that show each one fails its row:
  "restart_ignored"   the state after a done is the previous output, not the recorded one
  "zero_reset"        the state after a done is zero (R2D2's rule)
  "bptt_across_done"  the forward restarts, but the gradient flows into the previous step as if it had not
  "wgrad_recorded_h"  the W_h rows of the LSTM kernel gradient use the recorded h instead of h_in
  "wh_in_lstm_fwd"    the input GEMM still contracts the recorded h with W_h, on top of the recurrence
"""
import numpy as np
import torch

from oracle import impala_torch as it
from oracle import synthetic

import parity

BUGS = ("restart_ignored", "zero_reset", "bptt_across_done", "wgrad_recorded_h", "wh_in_lstm_fwd")


class RecurrentLearner(it.Learner):

    def __init__(self, params=None, dtype=torch.float64, bug=None, **cfg):
        super().__init__(params, dtype, "dedup", **cfg)
        if bug is not None and bug not in BUGS:
            raise ValueError(bug)
        self.bug = bug

    def _carry(self, d, h_prev, c_prev, h_rec, c_rec):
        d = d[:, None]
        if self.bug == "restart_ignored":
            return h_prev, c_prev
        if self.bug == "zero_reset":
            return torch.where(d, torch.zeros_like(h_prev), h_prev), torch.where(d, torch.zeros_like(c_prev), c_prev)
        if self.bug == "bptt_across_done":
            return (torch.where(d, h_rec + h_prev - h_prev.detach(), h_prev),
                    torch.where(d, c_rec + c_prev - c_prev.detach(), c_prev))
        return torch.where(d, h_rec, h_prev), torch.where(d, c_rec, c_prev)

    def _h_term(self, h, h_rec, Wh):
        if self.bug == "wgrad_recorded_h":      # value h W_h; dW_h from h_rec, dh from W_h
            return h @ Wh.detach() + h_rec @ Wh - (h_rec @ Wh).detach()
        if self.bug == "wh_in_lstm_fwd":
            return h @ Wh + h_rec @ Wh
        return h @ Wh

    def _unrolled(self, t):
        c, p = self.cfg, self.params
        T, A, L = c["trajectory"], c["num_action"], c["lstm_hidden_size"]
        B = t["x"].shape[0]
        img, conv = it.attention_cnn(p, t["x"].reshape(B * T, *t["x"].shape[2:]))
        emb = it.action_embedding(p, t["pa"].reshape(-1), A)
        x = torch.cat([img, emb], dim=1).reshape(B, T, -1)
        K = x.shape[2]
        Wx, Wh = p["lstm.w"][:K], p["lstm.w"][K:]
        h, cc = t["h0"][:, 0], t["c0"][:, 0]
        hin, cin, hout, cout = [], [], [], []
        for s in range(T):
            if s > 0:
                h, cc = self._carry(t["d"][:, s - 1], hout[-1], cout[-1], t["h0"][:, s], t["c0"][:, s])
            hin.append(h)
            cin.append(cc)
            z = x[:, s] @ Wx + self._h_term(h, t["h0"][:, s], Wh) + p["lstm.b"]
            i, j, f, o = torch.chunk(z, 4, dim=1)
            cc = torch.sigmoid(f + 1.0) * cc + torch.sigmoid(i) * torch.tanh(j)
            h = torch.sigmoid(o) * torch.tanh(cc)
            hout.append(h)
            cout.append(cc)
        h1 = torch.stack(hout, dim=1).reshape(B * T, L)
        logits = it.fully_connected(p, h1, "actor")
        pol = torch.softmax(logits, dim=1).reshape(B, T, A)
        val = it.fully_connected(p, h1, "critic").squeeze(1).reshape(B, T)
        taps = dict(a1=conv[0], a2=conv[1], a3=conv[2], emb=emb, logits=logits, policy=pol, value=val,
                    h1=h1.reshape(B, T, L), c1=torch.stack(cout, dim=1), hin=torch.stack(hin, dim=1),
                    cin=torch.stack(cin, dim=1))
        return (pol[:, :-2], val[:, :-2], pol[:, 1:-1], val[:, 1:-1], pol[:, 2:], val[:, 2:]), taps


def with_dones(batch, positions):
    """``batch`` with done set exactly at the (b, t) pairs of ``positions``."""
    out = dict(batch)
    d = np.zeros_like(batch["done"], dtype=bool)
    for b, t in positions:
        d[b, t] = True
    out["done"] = d
    return out


def default_dones(B, T):
    """Dones at several positions: t = 0, T - 1, the middle, adjacent pairs; several per trajectory."""
    pos = []
    for b in range(B):
        k = b % 4
        if k == 0:
            pos += [(b, 0), (b, T // 2)]
        elif k == 1:
            pos += [(b, T - 1), (b, 1), (b, 2)]
        elif k == 2:
            pos += [(b, T - 3), (b, T // 3)]
    return pos


def compare_step(B, T=20, A=18, seed=1234, steps=1, dones=None, **kw):
    """GPU recurrent learner against ``RecurrentLearner`` in float64 (at the GPU's ReLU pattern), as
    ``parity.compare_step``: {name: rel_err} for activations, the recurrence's buffers, V-trace taps, losses, every
    parameter gradient and the update / RMSProp slots after each of ``steps`` steps."""
    batch, params, cfg = parity.make_case(B, T, A, seed)
    batch = with_dones(batch, default_dones(B, T) if dones is None else dones)
    L = RecurrentLearner(params, **cfg)
    eng = parity.native_learner(batch, params, cfg, recurrent=True, **kw)
    args = [batch[k] for k in synthetic.TRAIN_FIELDS]
    M, Mb = B * T, B * (T - 2)
    errs = {}
    flips = elems = 0
    try:
        for s in range(steps):
            tag = "" if steps == 1 else "@%d" % s
            eng.stage(s % eng.num_slots, *args)
            out = eng.step(s % eng.num_slots)
            masks = parity.gpu_activation_pattern(eng, B, T, A)
            with it.activation_pattern(masks) as st:
                res, o, grads, gn = L.train(*args, return_all=True)
            flips, elems = flips + st["flips"], elems + st["elems"]
            for k in ("pi_loss", "baseline_loss", "entropy", "total_loss"):
                errs["loss/" + k + tag] = parity.rel_err(out[k], float(o[k].detach()))
            errs["grad_norm" + tag] = parity.rel_err(out["grad_norm"], gn)
            taps = eng.taps()
            for k in ("vs", "clipped_rho", "vs_plus_1", "pg_advantage"):
                errs["tap/" + k + tag] = parity.rel_err(taps[k], o[k].detach().numpy())
            gd = it.unflatten_params(eng.get_grads(), torch.float64, num_action=A)
            for n in grads:
                errs["grad/" + n + tag] = parity.rel_err(gd[n].numpy(), grads[n].detach().numpy())
            if s == 0:
                tp = o["taps"]
                errs["act/policy"] = parity.rel_err(eng.read_buffer("policy", M * A).reshape(M, A),
                                                    parity.to_time_major(tp["policy"].detach().numpy()))
                errs["act/value"] = parity.rel_err(eng.read_buffer("value", M),
                                                   parity.to_time_major(tp["value"].detach().numpy()))
                for dev, ref in (("hout", "h1"), ("c1", "c1"), ("hin", "hin"), ("cin", "cin")):
                    errs["act/" + dev] = parity.rel_err(eng.read_buffer(dev, M * 256).reshape(M, 256),
                                                        parity.to_time_major(tp[ref].detach().numpy()))
            pd = it.unflatten_params(eng.get_params(), torch.float64, num_action=A)
            for n in L.params:
                errs["param/" + n + tag] = parity.rel_err(pd[n].numpy(), L.params[n].detach().numpy())
        ms, _ = eng.get_opt_state()
        md = it.unflatten_params(ms, torch.float64, num_action=A)
        for n in L.params:
            errs["ms/" + n] = parity.rel_err(md[n].numpy(), L.ms[n].detach().numpy())
        errs["kink/flip_fraction"] = flips / max(elems, 1)
    finally:
        eng.close()
    return errs


def failures(errs, tol=parity.TOL):
    return {k: v for k, v in errs.items()
            if not v <= (parity.FLIP_FRACTION_MAX if k == "kink/flip_fraction" else tol)}
