"""PyTorch-CPU restatement of the reference IMPALA learner step -- TEST INFRASTRUCTURE ONLY.

float64 instance = truth for tolerances; float32 instance = "CPU restatement of the
reference, not TF1" timing baseline.  PINNED (see ``oracle/__init__.py``): ``tests/test_oracle_refexec.py`` executes the
unmodified ``agent/impala.py`` / ``model/impala_actor_critic.py`` over ``oracle/tf1_shim`` and this restatement equals it
(taps, losses, all gradients, three RMSProp steps) to ~1e-12 in float64.  The
TensorFlow 1.14 OP-KERNEL semantics shared by shim and restatement (conv2d VALID/NHWC/HWIO cross-correlation,
LSTMCell gate order i,j,f,o with forget_bias 1.0, RMSProp ms0=1 / eps inside sqrt,
clip_by_global_norm, polynomial_decay) are restated from SURVEY.md Appendix A.

Follows, line by line:
  model/impala_actor_critic.py:5-10   attention_CNN     -> ``attention_cnn``
  model/impala_actor_critic.py:12-16  action_embedding  -> ``action_embedding``
  model/impala_actor_critic.py:18-25  lstm              -> ``lstm``
  model/impala_actor_critic.py:27-30  fully_connected   -> ``fully_connected``
  model/impala_actor_critic.py:33-42  network           -> ``network``
  model/impala_actor_critic.py:44-118 build_network     -> ``build_network``
  agent/impala.py:31-100              graph             -> ``Learner.losses`` / ``Learner.train``
  agent/impala.py:132-148             Agent.train       -> ``Learner.train``
"""
import math
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------------------
# Parameter inventory (SURVEY.md App. A.6; TF1 variable creation order under
# {model_name}/impala/: conv2d, conv2d_1, conv2d_2, dense, dense_1, rnn/lstm_cell,
# dense_2..4 (actor), dense_5..7 (critic)).  Kernels in TF layouts: conv HWIO, dense [in,out].
# --------------------------------------------------------------------------------------
def param_specs(num_action=18, lstm_hidden_size=256, input_shape=(84, 84, 4)):
    h, w, c = input_shape
    o1 = ((h - 8) // 4 + 1, (w - 8) // 4 + 1)
    o2 = ((o1[0] - 4) // 2 + 1, (o1[1] - 4) // 2 + 1)
    o3 = (o2[0] - 3 + 1, o2[1] - 3 + 1)
    flat = o3[0] * o3[1] * 64
    L = lstm_hidden_size
    return [
        ("conv1.w", (8, 8, c, 32)), ("conv1.b", (32,)),
        ("conv2.w", (4, 4, 32, 64)), ("conv2.b", (64,)),
        ("conv3.w", (3, 3, 64, 64)), ("conv3.b", (64,)),
        ("emb1.w", (num_action, 256)), ("emb1.b", (256,)),
        ("emb2.w", (256, 256)), ("emb2.b", (256,)),
        ("lstm.w", (flat + 256 + L, 4 * L)), ("lstm.b", (4 * L,)),
        ("actor1.w", (L, 256)), ("actor1.b", (256,)),
        ("actor2.w", (256, 256)), ("actor2.b", (256,)),
        ("actor3.w", (256, num_action)), ("actor3.b", (num_action,)),
        ("critic1.w", (L, 256)), ("critic1.b", (256,)),
        ("critic2.w", (256, 256)), ("critic2.b", (256,)),
        ("critic3.w", (256, 1)), ("critic3.b", (1,)),
    ]


def param_count(**kw):
    return sum(int(np.prod(s)) for _, s in param_specs(**kw))


def init_params(seed=0, dtype=torch.float32, **kw):
    """glorot-uniform kernels (TF default for conv2d/dense/LSTMCell), zero biases.
    Generated in float32 from ``torch.Generator().manual_seed(seed)`` and cast, so the f64
    and f32 oracles and the GPU path all start from bit-identical float32 values."""
    g = torch.Generator().manual_seed(seed)
    out = OrderedDict()
    for name, shape in param_specs(**kw):
        if name.endswith(".b"):
            t = torch.zeros(shape, dtype=torch.float32)
        else:
            if len(shape) == 4:
                rf = shape[0] * shape[1]
                fan_in, fan_out = rf * shape[2], rf * shape[3]
            else:
                fan_in, fan_out = shape
            lim = math.sqrt(6.0 / (fan_in + fan_out))
            t = (torch.rand(shape, generator=g, dtype=torch.float32) * 2.0 - 1.0) * lim
        out[name] = t.to(dtype)
    return out


def flatten_params(params):
    """TF-layout tensors concatenated in ``param_specs`` order -> float32 numpy vector."""
    return np.concatenate([params[n].detach().to(torch.float32).reshape(-1).numpy()
                           for n in params]).astype(np.float32)


def unflatten_params(flat, dtype=torch.float32, **kw):
    out = OrderedDict()
    off = 0
    flat = np.asarray(flat)
    for name, shape in param_specs(**kw):
        n = int(np.prod(shape))
        out[name] = torch.from_numpy(np.array(flat[off:off + n], dtype=np.float32)).reshape(shape).to(dtype)
        off += n
    assert off == flat.size
    return out


# --------------------------------------------------------------------------------------
# Model (model/impala_actor_critic.py)
# --------------------------------------------------------------------------------------
def _conv2d_tf(x_nhwc, w_hwio, b, stride):
    """tf.layers.conv2d(padding='VALID', NHWC, kernel HWIO) = cross-correlation + bias."""
    y = F.conv2d(x_nhwc.permute(0, 3, 1, 2), w_hwio.permute(3, 2, 0, 1), b, stride=stride)
    return y.permute(0, 2, 3, 1)


# ReLU activation-pattern override (test aid).  ReLU' is discontinuous at 0: when a pre-activation is
# within float32 rounding of zero, a float32 implementation and this float64 oracle can legitimately
# disagree on the mask, and that single flip changes the gradient of the whole image by O(1e-3).
# ``activation_pattern(masks)`` makes the oracle evaluate relu(x) as x * mask with masks observed on the
# implementation under test (forward AND backward then follow the same branch) and records every
# element where sign(x) disagrees with the mask together with |x| there, so the caller can assert that
# flips are rare and only happen at |x| ~ 0.
_PATTERN = {"masks": None, "flips": 0, "elems": 0, "max_abs_at_flip": 0.0}


class activation_pattern:
    def __init__(self, masks):
        self.masks = masks

    def __enter__(self):
        _PATTERN.update(masks=self.masks, flips=0, elems=0, max_abs_at_flip=0.0)
        return _PATTERN

    def __exit__(self, *exc):
        _PATTERN["masks"] = None
        return False


def _relu(x, name, index=None):
    masks = _PATTERN["masks"]
    if masks is None or name not in masks:
        return F.relu(x)
    m = masks[name]
    if index is not None:
        m = m[index]
    m = m.reshape(x.shape).to(torch.bool)
    flip = (x > 0) != m
    n = int(flip.sum())
    _PATTERN["elems"] += x.numel()
    if n:
        _PATTERN["flips"] += n
        _PATTERN["max_abs_at_flip"] = max(_PATTERN["max_abs_at_flip"], float(x.detach().abs()[flip].max()))
    return x * m.to(x.dtype)


def attention_cnn(p, x):
    """model/impala_actor_critic.py:5-10; returns (flatten HWC, intermediates)."""
    a1 = _relu(_conv2d_tf(x, p["conv1.w"], p["conv1.b"], 4), "a1")
    a2 = _relu(_conv2d_tf(a1, p["conv2.w"], p["conv2.b"], 2), "a2")
    a3 = _relu(_conv2d_tf(a2, p["conv3.w"], p["conv3.b"], 1), "a3")
    return a3.reshape(a3.shape[0], -1), (a1, a2, a3)


def action_embedding(p, previous_action, num_action):
    """model/impala_actor_critic.py:12-16."""
    onehot = F.one_hot(previous_action.long(), num_action).to(p["emb1.w"].dtype)
    x = _relu(onehot @ p["emb1.w"] + p["emb1.b"], "e1", previous_action.long())
    return _relu(x @ p["emb2.w"] + p["emb2.b"], "emb", previous_action.long())


def lstm(p, inputs, initial_h, initial_c):
    """model/impala_actor_critic.py:18-25 -- one tf.nn.rnn_cell.LSTMCell step (TF 1.14):
    z=[x,h]W+b; i,j,f,o=split(z,4); c'=sig(f+1)*c+sig(i)*tanh(j); h'=sig(o)*tanh(c').
    Returns (output, c, h) like the reference (output == h')."""
    z = torch.cat([inputs, initial_h], dim=1) @ p["lstm.w"] + p["lstm.b"]
    i, j, f, o = torch.chunk(z, 4, dim=1)
    c = torch.sigmoid(f + 1.0) * initial_c + torch.sigmoid(i) * torch.tanh(j)
    h = torch.sigmoid(o) * torch.tanh(c)
    return h, c, h


def fully_connected(p, x, prefix):
    """model/impala_actor_critic.py:27-30 with hidden_list=[256,256]."""
    x = _relu(x @ p[prefix + "1.w"] + p[prefix + "1.b"], prefix + "1")
    x = _relu(x @ p[prefix + "2.w"] + p[prefix + "2.b"], prefix + "2")
    return x @ p[prefix + "3.w"] + p[prefix + "3.b"]


def network(p, image, previous_action, initial_h, initial_c, num_action, lstm_hidden_size,
            return_taps=False):
    """model/impala_actor_critic.py:33-42 -> (actor softmax, critic, c, h)."""
    image_embedding, conv_taps = attention_cnn(p, image)
    prev_emb = action_embedding(p, previous_action, num_action)
    concat = torch.cat([image_embedding, prev_emb], dim=1)
    out, c, h = lstm(p, concat, initial_h, initial_c)
    logits = fully_connected(p, out, "actor")
    actor = torch.softmax(logits, dim=1)
    critic = fully_connected(p, out, "critic").squeeze(1)
    if return_taps:
        return actor, critic, c, h, dict(a1=conv_taps[0], a2=conv_taps[1], a3=conv_taps[2],
                                         emb=prev_emb, logits=logits)
    return actor, critic, c, h


def build_network(p, state, previous_action, initial_h, initial_c,
                  trajectory_state, trajectory_previous_action,
                  trajectory_initial_h, trajectory_initial_c,
                  num_action, lstm_hidden_size, trajectory):
    """model/impala_actor_critic.py:44-118 -- REFERENCE-SHAPED: one single-step net plus
    3 x (T-2) per-timestep copies of ``network`` with shared weights."""
    policy, _, c, h = network(p, state, previous_action, initial_h, initial_c,
                              num_action, lstm_hidden_size)
    outs = []
    for lo, hi in ((0, -2), (1, -1), (2, None)):                         # first / middle / last
        ts = trajectory_state[:, lo:hi]
        tpa = trajectory_previous_action[:, lo:hi]
        th = trajectory_initial_h[:, lo:hi]
        tc = trajectory_initial_c[:, lo:hi]
        pol, val = [], []
        for i in range(trajectory - 2):
            a, v, _, _ = network(p, ts[:, i], tpa[:, i], th[:, i], tc[:, i],
                                 num_action, lstm_hidden_size)
            pol.append(a)
            val.append(v)
        outs += [torch.stack(pol, dim=1), torch.stack(val, dim=1)]
    return (policy, c, h, *outs)


# --------------------------------------------------------------------------------------
# V-trace in torch (optimizer/vtrace.py) -- same maths as oracle.vtrace_np, used so that
# autograd can differentiate the losses; the outputs are detached like tf.stop_gradient.
# --------------------------------------------------------------------------------------
def split_data(x):
    return x[:, :-2], x[:, 1:-1], x[:, 2:]


def _selected(softmax, actions):
    onehot = F.one_hot(actions.long(), softmax.shape[-1]).to(softmax.dtype)
    return torch.sum(softmax * onehot, dim=2)


def from_importance_weights(log_rhos, discounts, rewards, values, bootstrap_value,
                            clip_rho_threshold=1.0, clip_pg_rho_threshold=1.0):
    rhos = torch.exp(log_rhos)
    clipped_rhos = torch.clamp(rhos, max=clip_rho_threshold) if clip_rho_threshold is not None else rhos
    cs = torch.clamp(rhos, max=1.0)
    values_t_plus_1 = torch.cat([values[1:], bootstrap_value[None]], dim=0)
    deltas = clipped_rhos * (rewards + discounts * values_t_plus_1 - values)
    acc = torch.zeros_like(bootstrap_value)
    out = []
    for t in range(values.shape[0] - 1, -1, -1):
        acc = deltas[t] + discounts[t] * cs[t] * acc
        out.append(acc)
    vs = torch.stack(out[::-1], dim=0) + values
    return vs.detach(), clipped_rhos.detach()


def from_softmax(behavior_policy_softmax, target_policy_softmax, actions, discounts,
                 rewards, values, next_values, action_size, clip_rho_threshold=1.0,
                 clip_pg_rho_threshold=1.0):
    log_rhos = torch.log(_selected(target_policy_softmax, actions)) - \
        torch.log(_selected(behavior_policy_softmax, actions))
    vs, rho = from_importance_weights(log_rhos.t(), discounts.t(), rewards.t(), values.t(),
                                      next_values.t()[-1], clip_rho_threshold, clip_pg_rho_threshold)
    return vs.t(), rho.t()


def compute_policy_gradient_loss(softmax, actions, advantages, output_size):
    return -torch.sum(torch.log(_selected(softmax, actions) + 1e-8) * advantages.detach())


def compute_baseline_loss(vs, value):
    return torch.sum(torch.square(vs.detach() - value)) * 0.5


def compute_entropy_loss(softmax):
    return -torch.sum(torch.sum(-softmax * torch.log(softmax), dim=1))


def loss_inputs(reward, action, done, behavior_policy, dtype):
    """The fed tensors the losses read (agent/impala.py:134-142): r, a, d, mu."""
    return dict(r=torch.from_numpy(np.asarray(reward, dtype=np.float32)).to(dtype),
                a=torch.from_numpy(np.asarray(action).astype(np.int64)),
                d=torch.from_numpy(np.asarray(done).astype(bool)),
                mu=torch.from_numpy(np.asarray(behavior_policy, dtype=np.float32)).to(dtype))


def loss_terms(cfg, t, fp, fv, mp, mv, lp, lv):
    """agent/impala.py:45-93 from the first / middle / last policy [B, T-2, A] and value [B, T-2] windows and the
    prepared batch ``t`` (keys r, a, d, mu of ``loss_inputs``): V-trace targets, advantages and the three losses."""
    c = cfg
    if c["reward_clipping"] == "abs_one":                                # agent/impala.py:45-49
        cr = torch.clamp(t["r"], -1.0, 1.0)
    elif c["reward_clipping"] == "soft_asymmetric":
        sq = torch.tanh(t["r"] / 5.0)
        cr = torch.where(t["r"] < 0, 0.3 * sq, sq) * 5.0
    else:
        raise ValueError(c["reward_clipping"])
    discounts = (~t["d"]).to(fv.dtype) * c["discount_factor"]            # :51
    fa, ma, _ = split_data(t["a"])
    fr, mr, _ = split_data(cr)
    fd, md, _ = split_data(discounts)
    fb, mb, _ = split_data(t["mu"])
    A = c["num_action"]
    vs, clipped_rho = from_softmax(fb, fp, fa, fd, fr, fv, mv, A)          # :68-71
    vs_plus_1, _ = from_softmax(mb, mp, ma, md, mr, mv, lv, A)             # :73-76
    pg_adv = (clipped_rho * (fr + fd * vs_plus_1 - fv)).detach()          # :78-80
    pi_loss = compute_policy_gradient_loss(fp, fa, pg_adv, A)             # :82-86
    baseline_loss = compute_baseline_loss(vs, fv)                         # :87-89
    entropy = compute_entropy_loss(fp)                                    # :90-91
    total = pi_loss + baseline_loss * c["baseline_loss_coef"] + entropy * c["entropy_coef"]   # :93
    return dict(vs=vs, clipped_rho=clipped_rho, vs_plus_1=vs_plus_1, pg_advantage=pg_adv,
                pi_loss=pi_loss, baseline_loss=baseline_loss, entropy=entropy, total_loss=total,
                first_policy=fp, first_value=fv, middle_policy=mp, middle_value=mv,
                last_policy=lp, last_value=lv)


# --------------------------------------------------------------------------------------
# Learner (agent/impala.py)
# --------------------------------------------------------------------------------------
DEFAULT_CFG = dict(trajectory=20, input_shape=(84, 84, 4), num_action=18, lstm_hidden_size=256,
                   discount_factor=0.99, start_learning_rate=0.0006, end_learning_rate=0.0,
                   learning_frame=1000000000, baseline_loss_coef=1.0, entropy_coef=0.05,
                   gradient_clip_norm=40.0, reward_clipping="abs_one")   # config.json:130-143


def polynomial_decay_f32(start, step, decay_steps, end, power=1.0):
    """tf.train.polynomial_decay evaluated in float32 like the TF graph (dtype of learning_rate)."""
    gs = np.float32(min(float(step), float(decay_steps)))
    p = gs / np.float32(decay_steps)
    return np.float32((np.float32(start) - np.float32(end)) *
                      np.float32(np.power(np.float32(1.0) - p, np.float32(power))) + np.float32(end))


def global_norm(grads, dtype):
    """tf.global_norm of the gradient tensors ``grads``: the sum of squares is taken in float64 but overflows to inf
    where a ``dtype`` sum would (TF sums in the variables' float32), so the norm is inf exactly when TF's is."""
    ss = sum(torch.sum(v.double() ** 2) for v in grads)
    return torch.sqrt(ss).to(dtype) if bool(torch.isfinite(ss.to(dtype))) else ss.to(dtype)


def clip_scale(gn, clip):
    """The factor tf.clip_by_global_norm (TF 1.14 clip_ops) multiplies every gradient by:
    ``clip * min(1/norm, 1/clip) + (norm - norm)`` -- 1 for a zero norm, NaN for a NaN or infinite norm (TF's documented
    error signal: every clipped gradient becomes NaN)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        n = np.float64(gn)
        return float(clip * np.minimum(1.0 / n, 1.0 / clip) + (n - n))


class Learner:
    """agent/impala.py learner graph + Agent.train, on torch CPU.

    shaped='reference' executes the 54 per-timestep network copies + host float64 /255, as the
    reference graph does; shaped='dedup' evaluates the T distinct rows once (same maths, used
    for the big-batch parity cases).  RMSProp slots (ms0 = 1) and the step counter live here.
    """

    def __init__(self, params=None, dtype=torch.float32, shaped="dedup", **cfg):
        self.cfg = dict(DEFAULT_CFG)
        self.cfg.update(cfg)
        self.dtype = dtype
        self.shaped = shaped
        c = self.cfg
        kw = dict(num_action=c["num_action"], lstm_hidden_size=c["lstm_hidden_size"],
                  input_shape=tuple(c["input_shape"]))
        self._kw = kw
        if params is None:
            params = init_params(0, dtype, **kw)
        self.params = OrderedDict((k, v.detach().clone().to(dtype).requires_grad_(True))
                                  for k, v in params.items())
        self.ms = OrderedDict((k, torch.ones_like(v)) for k, v in self.params.items())
        self.step = 0

    # ---- inputs ------------------------------------------------------------------
    def _prep(self, state, reward, action, done, behavior_policy, previous_action, initial_h, initial_c):
        dt = self.dtype
        # agent/impala.py:133 -- float64 divide on the host, then the feed casts to float32.
        x = (np.stack(state).astype(np.float64) / 255).astype(np.float32)
        return dict(
            loss_inputs(reward, action, done, behavior_policy, dt),
            x=torch.from_numpy(x).to(dt),
            pa=torch.from_numpy(np.asarray(previous_action).astype(np.int64)),
            h0=torch.from_numpy(np.asarray(initial_h, dtype=np.float32)).to(dt),
            c0=torch.from_numpy(np.asarray(initial_c, dtype=np.float32)).to(dt))

    def _unrolled(self, t):
        """first/middle/last policy and value, [B, T-2, A] / [B, T-2]."""
        c, p = self.cfg, self.params
        T, A, L = c["trajectory"], c["num_action"], c["lstm_hidden_size"]
        B = t["x"].shape[0]
        if self.shaped == "reference":
            outs = build_network(p, t["x"][:, 0], t["pa"][:, 0], t["h0"][:, 0], t["c0"][:, 0],
                                 t["x"], t["pa"], t["h0"], t["c0"], A, L, T)
            return outs[3:], None
        # dedup: all B*T rows once; the three windows are slices (shift identity, App. C.4).
        pol, val, c1, h1, taps = network(p, t["x"].reshape(B * T, *t["x"].shape[2:]), t["pa"].reshape(-1),
                                         t["h0"].reshape(B * T, L), t["c0"].reshape(B * T, L), A, L,
                                         return_taps=True)
        pol = pol.reshape(B, T, A)
        val = val.reshape(B, T)
        taps = dict(taps, policy=pol, value=val, c1=c1.reshape(B, T, L), h1=h1.reshape(B, T, L))
        return (pol[:, :-2], val[:, :-2], pol[:, 1:-1], val[:, 1:-1], pol[:, 2:], val[:, 2:]), taps

    # ---- graph (agent/impala.py:45-93) -------------------------------------------
    def losses(self, state, reward, action, done, behavior_policy, previous_action, initial_h, initial_c):
        t = self._prep(state, reward, action, done, behavior_policy, previous_action, initial_h, initial_c)
        windows, taps = self._unrolled(t)
        return dict(loss_terms(self.cfg, t, *windows), taps=taps)

    def gradients(self, *batch, **kbatch):
        out = self.losses(*batch, **kbatch)
        names = list(self.params)
        extra = []
        if out.get("taps") is not None:          # also dL/d(activation) for the layer-wise parity diagnostics
            extra = [k for k in ("a1", "a2", "a3", "h1") if k in out["taps"]]
        grads = torch.autograd.grad(out["total_loss"], [self.params[n] for n in names] +
                                    [out["taps"][k] for k in extra], allow_unused=True)
        g = OrderedDict((n, (gi if gi is not None else torch.zeros_like(self.params[n])))
                        for n, gi in zip(names, grads))
        out["act_grads"] = {k: gi for k, gi in zip(extra, grads[len(names):])}
        return out, g

    # ---- Agent.train (agent/impala.py:95-100,132-148) ----------------------------
    def train(self, state, reward, action, done, behavior_policy, previous_action, initial_h, initial_c,
              return_all=False):
        c = self.cfg
        out, g = self.gradients(state, reward, action, done, behavior_policy, previous_action,
                                initial_h, initial_c)
        lr = polynomial_decay_f32(c["start_learning_rate"], self.step, c["learning_frame"],
                                  c["end_learning_rate"])                 # :96
        # tf.clip_by_global_norm: scale = clip * min(1/norm, 1/clip) + (norm - norm)
        gn = global_norm(g.values(), self.dtype)
        scale = clip_scale(gn, c["gradient_clip_norm"])
        with torch.no_grad():
            for n, p in self.params.items():                              # RMSProp(decay .99, eps .1)
                gc = g[n] * scale
                self.ms[n] += (gc * gc - self.ms[n]) * (1.0 - 0.99)
                p -= float(lr) * gc / torch.sqrt(self.ms[n] + 0.1)
        self.step += 1
        res = (float(out["pi_loss"].detach()), float(out["baseline_loss"].detach()), float(out["entropy"].detach()),
               float(lr))
        if return_all:
            return res, out, g, float(gn)
        return res

    def flat_params(self):
        return flatten_params(self.params)

    def flat_ms(self):
        return flatten_params(self.ms)


def flatten_grads(g):
    return np.concatenate([v.detach().to(torch.float64).reshape(-1).numpy() for v in g.values()])
