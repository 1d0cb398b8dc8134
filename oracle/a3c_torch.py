"""PyTorch-CPU restatement of the reference A3C learner step -- TEST INFRASTRUCTURE ONLY.  PINNED:
``tests/test_oracle_refexec.py`` executes the unmodified ``agent/a3c.py`` / ``model/actor_critic.py`` / ``optimizer/a2c.py`` over
``oracle/tf1_shim`` and this restatement equals it (policy, values, the three losses, all 22 gradients to ~1e-12, three Adam steps;
TensorFlow 1.14 itself is not installable here -- see ``oracle/__init__.py``); float64 = truth, float32 = CPU baseline.

Follows:
  model/actor_critic.py:3-39   attention_CNN / action_embedding / fully_connected / network -> ``network``
                               (the same layers as the Ape-X body; actor ends in softmax, critic is squeezed)
  model/actor_critic.py:41-56  build_network -> network(s, prev_a) and network(s', next_prev_a) with shared variables
  optimizer/a2c.py:3-26        compute_entropy_loss / compute_baseline_loss / compute_policy_loss -> same names
                               (policy loss uses the PROBABILITY pi(a), not its log; means over the batch)
  agent/a3c.py:36-81           graph + Adam(poly-decay lr) + clip_by_global_norm -> ``Learner.train``
  agent/a3c.py:85-103          Agent.train feeds next_previous_action = action
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

from . import apex_torch as ax
from . import impala_torch as it

BETA1, BETA2, ADAM_EPS = ax.BETA1, ax.BETA2, ax.ADAM_EPS


def param_specs(num_action=4, input_shape=(84, 84, 4)):
    """TF1 variable order under {model}/a3c: conv2d x3, dense x2 (embedding), dense x3 (actor), dense x3 (critic)."""
    ren = {"value": "actor", "mean": "critic"}
    out = []
    for name, shape in ax.param_specs(num_action=num_action, input_shape=input_shape):
        for k, v in ren.items():
            if name.startswith(k):
                name = v + name[len(k):]
        out.append((name, shape))
    return out


def param_count(**kw):
    return sum(int(np.prod(s)) for _, s in param_specs(**kw))


def init_params(seed=0, dtype=torch.float32, **kw):
    p = ax.init_params(seed, dtype, **kw)
    return OrderedDict((n, v) for (n, _), v in zip(param_specs(**kw), p.values()))


flatten_params = ax.flatten_params


def unflatten_params(flat, dtype=torch.float32, **kw):
    out, off = OrderedDict(), 0
    flat = np.asarray(flat)
    for name, shape in param_specs(**kw):
        n = int(np.prod(shape))
        out[name] = torch.from_numpy(np.array(flat[off:off + n], dtype=np.float32)).reshape(shape).to(dtype)
        off += n
    assert off == flat.size
    return out


def network(p, image, previous_action, num_action, return_taps=False):
    """model/actor_critic.py:28-39 -> (actor softmax [N,A], critic [N])."""
    emb_img, conv = it.attention_cnn(p, image)
    emb_a = it.action_embedding(p, previous_action, num_action)
    concat = torch.cat([emb_img, emb_a], dim=1)
    actor = torch.softmax(it.fully_connected(p, concat, "actor"), dim=1)
    critic = it.fully_connected(p, concat, "critic").squeeze(1)
    if return_taps:
        return actor, critic, dict(a1=conv[0], a2=conv[1], a3=conv[2])
    return actor, critic


def compute_entropy_loss(policy):                                   # optimizer/a2c.py:3-7
    return -torch.mean(torch.sum(-policy * torch.log(policy), dim=1))


def compute_baseline_loss(value, next_value, discounts, reward):    # optimizer/a2c.py:9-15
    diff = reward + discounts * next_value.detach() - value
    return torch.mean(diff * diff)


def compute_policy_loss(policy, action, value, next_value, discounts, reward, num_action):   # optimizer/a2c.py:17-26
    sel = torch.sum(policy * F.one_hot(action.long(), num_action).to(policy.dtype), dim=1)
    adv = (reward + discounts * next_value - value).detach()
    return -torch.mean(adv * sel)


DEFAULT_CFG = dict(input_shape=(84, 84, 4), num_action=4, discount_factor=0.997, start_learning_rate=1e-4,
                   end_learning_rate=0.0, learning_frame=1000000000, baseline_loss_coef=1.0, entropy_coef=0.05,
                   gradient_clip_norm=40.0, reward_clipping="abs_one")          # config.json:2-41


class Learner:
    def __init__(self, params=None, dtype=torch.float32, **cfg):
        self.cfg = dict(DEFAULT_CFG)
        self.cfg.update(cfg)
        self.dtype = dtype
        c = self.cfg
        self._kw = dict(num_action=c["num_action"], input_shape=tuple(c["input_shape"]))
        if params is None:
            params = init_params(0, dtype, **self._kw)
        self.params = OrderedDict((k, v.detach().clone().to(dtype).requires_grad_(True)) for k, v in params.items())
        self.m = OrderedDict((k, torch.zeros_like(v)) for k, v in self.params.items())
        self.v = OrderedDict((k, torch.zeros_like(v)) for k, v in self.params.items())
        self.beta1_power, self.beta2_power = np.float32(BETA1), np.float32(BETA2)
        self.step = 0

    def _img(self, s):
        return torch.from_numpy((np.stack(s).astype(np.float64) / 255).astype(np.float32)).to(self.dtype)

    def policy_value(self, state, previous_action):
        with torch.no_grad():
            return network(self.params, self._img(state), torch.from_numpy(np.asarray(previous_action).astype(np.int64)),
                           self.cfg["num_action"])

    def losses(self, state, next_state, previous_action, action, reward, done):
        c = self.cfg
        A = c["num_action"]
        pa = torch.from_numpy(np.asarray(previous_action).astype(np.int64))
        a = torch.from_numpy(np.asarray(action).astype(np.int64))
        r = torch.from_numpy(np.asarray(reward, dtype=np.float32)).to(self.dtype)
        d = torch.from_numpy(np.asarray(done).astype(bool))
        if c["reward_clipping"] == "abs_one":                                            # agent/a3c.py:38-43
            cr = torch.clamp(r, -1.0, 1.0)
        else:
            sq = torch.tanh(r / 5.0)
            cr = torch.where(r < 0, 0.3 * sq, sq) * 5.0
        discounts = (~d).to(self.dtype) * c["discount_factor"]
        policy, value, taps = network(self.params, self._img(state), pa, A, return_taps=True)
        with torch.no_grad():
            saved = it._PATTERN["masks"]
            it._PATTERN["masks"] = None
            try:
                _, next_value = network(self.params, self._img(next_state), a, A)      # agent/a3c.py:99: npa = action
            finally:
                it._PATTERN["masks"] = saved
        pi = compute_policy_loss(policy, a, value, next_value, discounts, cr, A)
        bl = compute_baseline_loss(value, next_value, discounts, cr)
        en = compute_entropy_loss(policy)
        total = pi + bl * c["baseline_loss_coef"] + en * c["entropy_coef"]
        return dict(policy=policy, value=value, next_value=next_value, advantage=(cr + discounts * next_value - value).detach(),
                    pi_loss=pi, baseline_loss=bl, entropy=en, total_loss=total, taps=taps)

    def train(self, state, next_state, previous_action, action, reward, done, return_all=False):
        c = self.cfg
        out = self.losses(state, next_state, previous_action, action, reward, done)
        names = list(self.params)
        grads = torch.autograd.grad(out["total_loss"], [self.params[n] for n in names], allow_unused=True)
        g = OrderedDict((n, (gi if gi is not None else torch.zeros_like(self.params[n]))) for n, gi in zip(names, grads))
        lr = it.polynomial_decay_f32(c["start_learning_rate"], self.step, c["learning_frame"], c["end_learning_rate"])
        gn = it.global_norm(g.values(), self.dtype)
        scale = it.clip_scale(gn, c["gradient_clip_norm"])
        alpha = float(lr) * np.sqrt(1.0 - float(self.beta2_power)) / (1.0 - float(self.beta1_power))
        with torch.no_grad():
            for n, p in self.params.items():
                gc = g[n] * scale
                self.m[n] += (gc - self.m[n]) * (1.0 - BETA1)
                self.v[n] += (gc * gc - self.v[n]) * (1.0 - BETA2)
                p -= self.m[n] * alpha / (torch.sqrt(self.v[n]) + ADAM_EPS)
        self.beta1_power = np.float32(self.beta1_power * np.float32(BETA1))
        self.beta2_power = np.float32(self.beta2_power * np.float32(BETA2))
        self.step += 1
        res = (float(out["pi_loss"].detach().item()), float(out["baseline_loss"].detach().item()),
               float(out["entropy"].detach().item()), float(lr))
        if return_all:
            return res, out, g, float(gn)
        return res


TRAIN_FIELDS = ("state", "next_state", "previous_action", "action", "reward", "done")
make_transitions = ax.make_transitions
