"""PyTorch-CPU restatement of the reference R2D2 learner step -- TEST INFRASTRUCTURE ONLY.

float64 instance = truth for tolerances; float32 instance = "CPU restatement of the reference, not TF1" timing
baseline.  PINNED (see ``oracle/__init__.py``): ``tests/test_oracle_refexec.py`` executes the unmodified ``agent/r2d2.py`` /
``model/r2d2_lstm.py`` / ``optimizer/burn_in.py`` over ``oracle/tf1_shim`` and this restatement equals it in float64.  TensorFlow 1.14
itself is not installable here; TF OP-KERNEL semantics (LSTMCell gate order i,j,f,o with forget_bias 1.0, dynamic_rnn over a
length-1 sequence from a fed (c, h) state, AdamOptimizer.minimize = ApplyAdam without clipping) restated from
the TF 1.14 documentation.

Follows, line by line:
  model/r2d2_lstm.py:28-53    network        -> ``network`` (3 convs, action embedding, concat, ONE LSTMCell step,
                                                dense 128 ReLU, value [A] and a separate "mean" [1] stream, q = value - mean)
  model/r2d2_lstm.py:55-116   build_network  -> ``unroll``: seq_len truly recurrent steps per scope; after step i the
                                                carried (h, c) are multiplied by (1 - done_i) (:79-81, :108-110); the q of
                                                step i is computed from the UN-masked output
  optimizer/burn_in.py:23-32  value_function_rescaling / inverse_value_function_rescaling -> ``vf_rescale`` / ``vf_rescale_inv``
  agent/r2d2.py:62-90         graph          -> ``Learner.losses`` (burn-in slices the LOSS window only: gradients still
                                                flow through the burn-in steps; rewards are NOT clipped here)
  agent/r2d2.py:91-92         Adam(1e-4).minimize -> ``Learner.train``
  agent/r2d2.py:97-130        get_td_error   -> ``Learner.get_td_error`` (|mean over the whole window of target - q|)
  agent/r2d2.py:132-159       train          -> ``Learner.train`` -> (loss, |mean_t(target - q)| per sequence)
  agent/r2d2.py:164-165       main_to_target -> ``Learner.main_to_target`` (target <- main, utils.py:27-32)
  agent/r2d2.py:171-191       get_action     -> ``Learner.step_q``
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

from . import impala_torch as it

BETA1, BETA2, ADAM_EPS, LR = 0.9, 0.999, 1e-8, 1e-4          # tf.train.AdamOptimizer(learning_rate=1e-4) defaults
EPS_RESCALE = 1e-3                                           # agent/r2d2.py:85,88


def param_specs(num_action=4, lstm_size=64, input_shape=(84, 84, 1)):
    """TF1 variable-creation order under {model}/main/ (and again under {model}/target/): conv2d x3, dense, dense_1
    (action embedding), rnn/lstm_cell/{kernel,bias}, dense_2 (128), dense_3 (value), dense_4 (mean)."""
    h, w, c = input_shape
    o1 = ((h - 8) // 4 + 1, (w - 8) // 4 + 1)
    o2 = ((o1[0] - 4) // 2 + 1, (o1[1] - 4) // 2 + 1)
    o3 = (o2[0] - 2, o2[1] - 2)
    cat = o3[0] * o3[1] * 64 + 256
    L = lstm_size
    return [("conv1.w", (8, 8, c, 32)), ("conv1.b", (32,)), ("conv2.w", (4, 4, 32, 64)), ("conv2.b", (64,)),
            ("conv3.w", (3, 3, 64, 64)), ("conv3.b", (64,)), ("emb1.w", (num_action, 256)), ("emb1.b", (256,)),
            ("emb2.w", (256, 256)), ("emb2.b", (256,)), ("lstm.w", (cat + L, 4 * L)), ("lstm.b", (4 * L,)),
            ("q1.w", (L, 128)), ("q1.b", (128,)), ("value.w", (128, num_action)), ("value.b", (num_action,)),
            ("mean.w", (128, 1)), ("mean.b", (1,))]


def param_count(**kw):
    return sum(int(np.prod(s)) for _, s in param_specs(**kw))


def init_params(seed=0, dtype=torch.float32, **kw):
    import math
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
    return np.concatenate([params[n].detach().to(torch.float32).reshape(-1).numpy() for n in params]).astype(np.float32)


def unflatten_params(flat, dtype=torch.float32, **kw):
    out, off = OrderedDict(), 0
    flat = np.asarray(flat)
    for name, shape in param_specs(**kw):
        n = int(np.prod(shape))
        out[name] = torch.from_numpy(np.array(flat[off:off + n], dtype=np.float32)).reshape(shape).to(dtype)
        off += n
    assert off == flat.size
    return out


def vf_rescale(x, eps=EPS_RESCALE):
    """optimizer/burn_in.py:23-25: sign(x)(sqrt(|x| + 1) - 1) + eps x."""
    return torch.sign(x) * (torch.sqrt(torch.abs(x) + 1.0) - 1.0) + eps * x


def vf_rescale_inv(x, eps=EPS_RESCALE):
    """optimizer/burn_in.py:27-32: sign(x)(((sqrt(1 + 4 eps (|x| + 1 + eps)) - 1) / (2 eps))^2 - 1)."""
    return torch.sign(x) * (torch.square((torch.sqrt(1.0 + 4.0 * eps * (torch.abs(x) + 1.0 + eps)) - 1.0) / (2.0 * eps)) - 1.0)


def network(p, state, previous_action, h, c, num_action, t=None):
    """model/r2d2_lstm.py:28-53 -> (q [N,A], h', c').  `t` only indexes the ReLU pattern override of a time step."""
    def relu(x, name):
        return it._relu(x, name, t) if t is not None else it._relu(x, name)
    a1 = relu(it._conv2d_tf(state, p["conv1.w"], p["conv1.b"], 4), "a1")
    a2 = relu(it._conv2d_tf(a1, p["conv2.w"], p["conv2.b"], 2), "a2")
    a3 = relu(it._conv2d_tf(a2, p["conv3.w"], p["conv3.b"], 1), "a3")
    flat = a3.reshape(a3.shape[0], -1)
    emb = it.action_embedding(p, previous_action, num_action)
    x = torch.cat([flat, emb], dim=1)
    z = torch.cat([x, h], dim=1) @ p["lstm.w"] + p["lstm.b"]          # TF LSTMCell: [inputs, h] @ kernel
    i, j, f, o = torch.chunk(z, 4, dim=1)
    c2 = torch.sigmoid(f + 1.0) * c + torch.sigmoid(i) * torch.tanh(j)
    h2 = torch.sigmoid(o) * torch.tanh(c2)
    q1 = relu(h2 @ p["q1.w"] + p["q1.b"], "q1")
    value = q1 @ p["value.w"] + p["value.b"]
    mean = q1 @ p["mean.w"] + p["mean.b"]
    return value - mean, h2, c2, dict(a1=a1, a2=a2, a3=a3)


def unroll(p, state, previous_action, done, h0, c0, num_action, pattern=False):
    """model/r2d2_lstm.py:67-84 -> q [B, S, A] (+ per-step conv activations when `pattern`)."""
    S = state.shape[1]
    h, c = h0, c0
    qs, taps = [], []
    for i in range(S):
        q, h, c, tp = network(p, state[:, i], previous_action[:, i], h, c, num_action, t=i if pattern else None)
        qs.append(q)
        taps.append(tp)
        keep = (~done[:, i]).to(q.dtype).unsqueeze(1)
        h, c = h * keep, c * keep
    return torch.stack(qs, dim=1), taps


DEFAULT_CFG = dict(seq_len=15, burn_in=7, input_shape=(84, 84, 1), num_action=4, lstm_size=64,
                   discount_factor=0.997, learning_rate=LR)    # config.json:84-101; agent/r2d2.py's fixed Adam rate


class Learner:
    def __init__(self, params=None, target_params=None, dtype=torch.float32, **cfg):
        self.cfg = dict(DEFAULT_CFG)
        self.cfg.update(cfg)
        self.dtype = dtype
        c = self.cfg
        self._kw = dict(num_action=c["num_action"], lstm_size=c["lstm_size"], input_shape=tuple(c["input_shape"]))
        if params is None:
            params = init_params(0, dtype, **self._kw)
        if target_params is None:
            target_params = init_params(1, dtype, **self._kw)
        self.params = OrderedDict((k, v.detach().clone().to(dtype).requires_grad_(True)) for k, v in params.items())
        self.target = OrderedDict((k, v.detach().clone().to(dtype)) for k, v in target_params.items())
        self.m = OrderedDict((k, torch.zeros_like(v)) for k, v in self.params.items())
        self.v = OrderedDict((k, torch.zeros_like(v)) for k, v in self.params.items())
        self.beta1_power, self.beta2_power = np.float32(BETA1), np.float32(BETA2)
        self.step = 0

    def main_to_target(self):
        with torch.no_grad():
            for k in self.target:
                self.target[k] = self.params[k].detach().clone()

    def _img(self, s):
        return torch.from_numpy((np.stack(s).astype(np.float64) / 255).astype(np.float32)).to(self.dtype)

    def step_q(self, state, h, c, previous_action):
        """agent/r2d2.py:171-181 (batched): -> (q [n,A], h' [n,L], c' [n,L])."""
        with torch.no_grad():
            q, h2, c2, _ = network(self.params, self._img(state), torch.from_numpy(np.asarray(previous_action).astype(np.int64)),
                                   torch.from_numpy(np.asarray(h, np.float32)).to(self.dtype),
                                   torch.from_numpy(np.asarray(c, np.float32)).to(self.dtype), self.cfg["num_action"])
        return q.numpy(), h2.numpy(), c2.numpy()

    def losses(self, state, previous_action, action, h, c, reward, done, weight=None, next_action=None):
        """agent/r2d2.py:62-90.  h, c: [B, S, L] as stored by the actors; only [:, 0] is fed (:140-141)."""
        cf = self.cfg
        A, bi = cf["num_action"], cf["burn_in"]
        x = self._img(state)
        pa = torch.from_numpy(np.asarray(previous_action).astype(np.int64))
        a = torch.from_numpy(np.asarray(action).astype(np.int64))
        r = torch.from_numpy(np.asarray(reward, dtype=np.float32)).to(self.dtype)
        d = torch.from_numpy(np.asarray(done).astype(bool))
        h0 = torch.from_numpy(np.asarray(h, np.float32)[:, 0]).to(self.dtype)
        c0 = torch.from_numpy(np.asarray(c, np.float32)[:, 0]).to(self.dtype)
        B = x.shape[0]
        w = torch.ones(B, dtype=self.dtype) if weight is None else torch.from_numpy(np.asarray(weight, np.float32)).to(self.dtype)
        main_q, taps = unroll(self.params, x, pa, d, h0, c0, A, pattern=it._PATTERN["masks"] is not None)
        with torch.no_grad():
            saved = it._PATTERN["masks"]
            it._PATTERN["masks"] = None
            try:
                target_q, _ = unroll(self.target, x, pa, d, h0, c0, A)
            finally:
                it._PATTERN["masks"] = saved
        discounts = (~d).to(self.dtype) * cf["discount_factor"]                         # :62
        bm, bt = main_q[:, bi:], target_q[:, bi:]                                       # :64-68
        state_main_q, next_main_q, next_target_q = bm[:, :-1], bm[:, 1:], bt[:, 1:]     # :70-72
        act, rew, disc = a[:, bi:][:, :-1], r[:, bi:][:, :-1], discounts[:, bi:][:, :-1]
        if next_action is None:
            next_action = torch.argmax(next_main_q, dim=2)                              # :74
        else:
            next_action = torch.from_numpy(np.asarray(next_action).astype(np.int64))
        sav = torch.sum(state_main_q * F.one_hot(act, A).to(self.dtype), dim=2)          # :81
        nsav = torch.sum(next_target_q * F.one_hot(next_action, A).to(self.dtype), dim=2)
        rescaled_target = (vf_rescale_inv(nsav) * disc + rew).detach()                  # :83-86
        target_value = vf_rescale(rescaled_target)                                      # :87-88
        unweighted = torch.mean((target_value - sav) ** 2, dim=1)                       # :89
        value_loss = torch.mean(unweighted * w)                                         # :90
        return dict(main_q=main_q, target_q=target_q, next_action=next_action, state_action_value=sav,
                    target_value=target_value, value_loss=value_loss, taps=taps)

    def get_td_error(self, state, previous_action, action, h, c, reward, done):
        """agent/r2d2.py:97-130 for ONE sequence -> scalar |mean(target_value - state_action_value)|."""
        with torch.no_grad():
            o = self.losses([state], [previous_action], [action], [h], [c], [reward], [done])
        return float(np.abs(np.mean(o["target_value"].numpy() - o["state_action_value"].numpy())))

    def gradients(self, *batch, **kw):
        out = self.losses(*batch, **kw)
        names = list(self.params)
        grads = torch.autograd.grad(out["value_loss"], [self.params[n] for n in names], allow_unused=True)
        g = OrderedDict((n, (gi if gi is not None else torch.zeros_like(self.params[n]))) for n, gi in zip(names, grads))
        return out, g

    def train(self, state, previous_action, action, h, c, reward, done, weight, return_all=False, next_action=None):
        """agent/r2d2.py:132-159 -> (loss, td_error [B]) from BEFORE the update."""
        out, g = self.gradients(state, previous_action, action, h, c, reward, done, weight=weight,
                                next_action=next_action)
        b1p, b2p = float(self.beta1_power), float(self.beta2_power)
        alpha = float(np.float32(self.cfg["learning_rate"])) * np.sqrt(1.0 - b2p) / (1.0 - b1p)
        with torch.no_grad():
            for n, p in self.params.items():
                self.m[n] += (g[n] - self.m[n]) * (1.0 - BETA1)
                self.v[n] += (g[n] * g[n] - self.v[n]) * (1.0 - BETA2)
                p -= self.m[n] * alpha / (torch.sqrt(self.v[n]) + ADAM_EPS)
        self.beta1_power = np.float32(self.beta1_power * np.float32(BETA1))
        self.beta2_power = np.float32(self.beta2_power * np.float32(BETA2))
        self.step += 1
        diff = out["target_value"].numpy() - out["state_action_value"].detach().numpy()
        td = np.abs(np.mean(diff, axis=1))
        res = (float(out["value_loss"].detach().item()), td)
        if return_all:
            gn = float(torch.sqrt(sum(torch.sum(v.double() ** 2) for v in g.values())))
            return res, out, g, gn
        return res


def make_sequences(B, S=15, A=4, L=64, input_shape=(84, 84, 1), seed=2468):
    """Seeded synthetic R2D2 minibatch: the fields train_r2d2.py:139-159 feeds (state uint8 [B,S,84,84,C];
    previous_action, action int32 [B,S]; h, c float32 [B,S,L] (only [:,0] is used); reward float32; done bool; weight)."""
    rng = np.random.default_rng(seed)
    state = rng.integers(0, 256, (B, S, *input_shape), dtype=np.uint8)
    previous_action = rng.integers(0, A, (B, S)).astype(np.int32)
    action = rng.integers(0, A, (B, S)).astype(np.int32)
    h = np.clip(rng.standard_normal((B, S, L)) * 0.5, -0.999, 0.999).astype(np.float32)
    c = rng.standard_normal((B, S, L)).astype(np.float32)
    reward = rng.standard_normal((B, S)).astype(np.float32)
    reward[rng.random((B, S)) < 0.3] = 0.0
    done = rng.random((B, S)) < 0.08
    weight = rng.uniform(0.2, 1.0, (B,)).astype(np.float32)
    weight[rng.integers(0, B)] = 1.0
    return dict(state=state, previous_action=previous_action, action=action, h=h, c=c, reward=reward, done=done,
                weight=weight)


TRAIN_FIELDS = ("state", "previous_action", "action", "h", "c", "reward", "done", "weight")
