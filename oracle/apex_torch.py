"""PyTorch-CPU restatement of the reference Ape-X DQN learner step -- TEST INFRASTRUCTURE ONLY.

float64 instance = truth for tolerances; float32 instance = "CPU restatement of the reference, not
TF1" timing baseline.  PINNED (see ``oracle/__init__.py``): ``tests/test_oracle_refexec.py`` executes the unmodified
``agent/apex.py`` / ``model/apex_value.py`` over ``oracle/tf1_shim`` and this restatement equals it (q values, loss, |td|,
Adam steps, target sync) in float64.  TensorFlow 1.14 itself is not
installable here; the TF OP-KERNEL semantics (conv2d VALID/NHWC/HWIO,
AdamOptimizer's ApplyAdam, clip_by_global_norm with ``None`` gradients skipped, polynomial_decay in
float32, tf.argmax = first maximal index) are restated from the TF 1.14 documentation.

Follows, line by line:
  model/apex_value.py:4-9     attention_CNN      -> ``oracle.impala_torch.attention_cnn`` (same layers)
  model/apex_value.py:11-15   action_embedding   -> ``oracle.impala_torch.action_embedding``
  model/apex_value.py:17-20   fully_connected    -> ``oracle.impala_torch.fully_connected``
  model/apex_value.py:22-41   dueling_network    -> ``dueling_network`` (q = value - mean, where "mean"
                                                   is a SEPARATE dense(.., 1) head, not mean-of-advantages)
  model/apex_value.py:43-66   build_network      -> ``Learner.q_values`` (main(s, prev_a), main(s', a), target(s', a))
  optimizer/dqn.py:3-7        take_state_action_value -> ``take_state_action_value``
  agent/apex.py:30-68         graph              -> ``Learner.losses``
  agent/apex.py:70-75         Adam train op      -> ``Learner.distributed_train``
  agent/apex.py:78-79         target_to_main     -> ``Learner.target_to_main`` (copies MAIN INTO TARGET, despite the name:
                                                   utils.py:27-32 zips get_vars('.../main') with get_vars('.../target') and
                                                   assigns v_targ <- v_main; the Adam slots that also match '.../main' come
                                                   later in tf.global_variables() and are cut off by zip)
  agent/apex.py:88-102        get_policy_and_action -> ``Learner.main_q``
  agent/apex.py:116-133       get_td_error       -> ``Learner.get_td_error``
  agent/apex.py:135-154       distributed_train  -> ``Learner.distributed_train``
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

from . import impala_torch as it


# --------------------------------------------------------------------------------------
# Parameter inventory: TF1 variable creation order under {model_name}/main/ (and the same again under
# {model_name}/target/): conv2d, conv2d_1, conv2d_2, dense, dense_1 (action embedding), dense_2..4
# (value stream 3392 -> 256 -> 256 -> A), dense_5..7 ("mean" stream 3392 -> 256 -> 256 -> 1).
# --------------------------------------------------------------------------------------
def param_specs(num_action=4, input_shape=(84, 84, 4), hidden=256):
    h, w, c = input_shape
    o1 = ((h - 8) // 4 + 1, (w - 8) // 4 + 1)
    o2 = ((o1[0] - 4) // 2 + 1, (o1[1] - 4) // 2 + 1)
    o3 = (o2[0] - 3 + 1, o2[1] - 3 + 1)
    flat = o3[0] * o3[1] * 64
    cat = flat + 256
    return [
        ("conv1.w", (8, 8, c, 32)), ("conv1.b", (32,)),
        ("conv2.w", (4, 4, 32, 64)), ("conv2.b", (64,)),
        ("conv3.w", (3, 3, 64, 64)), ("conv3.b", (64,)),
        ("emb1.w", (num_action, 256)), ("emb1.b", (256,)),
        ("emb2.w", (256, 256)), ("emb2.b", (256,)),
        ("value1.w", (cat, hidden)), ("value1.b", (hidden,)),
        ("value2.w", (hidden, hidden)), ("value2.b", (hidden,)),
        ("value3.w", (hidden, num_action)), ("value3.b", (num_action,)),
        ("mean1.w", (cat, hidden)), ("mean1.b", (hidden,)),
        ("mean2.w", (hidden, hidden)), ("mean2.b", (hidden,)),
        ("mean3.w", (hidden, 1)), ("mean3.b", (1,)),
    ]


def param_count(**kw):
    return sum(int(np.prod(s)) for _, s in param_specs(**kw))


def init_params(seed=0, dtype=torch.float32, **kw):
    """glorot-uniform kernels, zero biases (tf.layers defaults), float32 values from a seeded generator."""
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
# Model (model/apex_value.py)
# --------------------------------------------------------------------------------------
def dueling_network(p, image, previous_action, num_action, return_taps=False):
    """model/apex_value.py:22-41 -> q_value [N, A] = value_stream - mean_stream."""
    image_embedding, conv_taps = it.attention_cnn(p, image)
    prev_emb = it.action_embedding(p, previous_action, num_action)
    concat = torch.cat([image_embedding, prev_emb], dim=1)
    value = it.fully_connected(p, concat, "value")
    mean = it.fully_connected(p, concat, "mean")
    q = value - mean
    if return_taps:
        return q, dict(a1=conv_taps[0], a2=conv_taps[1], a3=conv_taps[2], emb=prev_emb, value=value, mean=mean)
    return q


def take_state_action_value(state_value, action, num_action):
    """optimizer/dqn.py:3-7."""
    onehot = F.one_hot(action.long(), num_action).to(state_value.dtype)
    return torch.sum(state_value * onehot, dim=1)


DEFAULT_CFG = dict(input_shape=(84, 84, 4), num_action=4, discount_factor=0.99, gradient_clip_norm=40.0,
                   reward_clipping="abs_one", start_learning_rate=1e-4, end_learning_rate=0.0,
                   learning_frame=100000000000000)          # config.json:146-184

BETA1, BETA2, ADAM_EPS = 0.9, 0.999, 1e-8                   # tf.train.AdamOptimizer defaults (agent/apex.py:72)


class Learner:
    """agent/apex.py learner graph + distributed_train / get_td_error / train, on torch CPU."""

    def __init__(self, params=None, target_params=None, dtype=torch.float32, **cfg):
        self.cfg = dict(DEFAULT_CFG)
        self.cfg.update(cfg)
        self.dtype = dtype
        c = self.cfg
        self._kw = dict(num_action=c["num_action"], input_shape=tuple(c["input_shape"]))
        if params is None:
            params = init_params(0, dtype, **self._kw)
        if target_params is None:
            target_params = init_params(1, dtype, **self._kw)     # TF initialises 'target' independently of 'main'
        self.params = OrderedDict((k, v.detach().clone().to(dtype).requires_grad_(True)) for k, v in params.items())
        self.target = OrderedDict((k, v.detach().clone().to(dtype)) for k, v in target_params.items())
        self.m = OrderedDict((k, torch.zeros_like(v)) for k, v in self.params.items())
        self.v = OrderedDict((k, torch.zeros_like(v)) for k, v in self.params.items())
        self.beta1_power = np.float32(BETA1)     # float32 non-trainable variables, multiplied after every apply
        self.beta2_power = np.float32(BETA2)
        self.step = 0

    def target_to_main(self):
        """agent/apex.py:78-79 + utils.py:27-32: target <- main."""
        with torch.no_grad():
            for k in self.target:
                self.target[k] = self.params[k].detach().clone()

    # ---- inputs ------------------------------------------------------------------
    def _img(self, s):
        # agent/apex.py:117-118,137-138: np.stack(state) / 255 in float64, cast to float32 at the feed
        return torch.from_numpy((np.stack(s).astype(np.float64) / 255).astype(np.float32)).to(self.dtype)

    def main_q(self, state, previous_action):
        """agent/apex.py:88-96 (batched): main_q_value for n states."""
        with torch.no_grad():
            return dueling_network(self.params, self._img(state),
                                   torch.from_numpy(np.asarray(previous_action).astype(np.int64)),
                                   self.cfg["num_action"])

    # ---- graph (agent/apex.py:30-68) -------------------------------------------------
    def losses(self, state, next_state, previous_action, action, reward, done, is_weight=None, next_action=None):
        """``next_action`` (test aid) overrides argmax(next_main_q): where the two largest q-values of a row are
        within float32 rounding, a float32 implementation may legitimately pick the other one."""
        c = self.cfg
        A = c["num_action"]
        x, nx = self._img(state), self._img(next_state)
        pa = torch.from_numpy(np.asarray(previous_action).astype(np.int64))
        a = torch.from_numpy(np.asarray(action).astype(np.int64))
        r = torch.from_numpy(np.asarray(reward, dtype=np.float32)).to(self.dtype)
        d = torch.from_numpy(np.asarray(done).astype(bool))
        if is_weight is None:
            w = torch.ones_like(r)
        else:
            w = torch.from_numpy(np.asarray(is_weight, dtype=np.float32)).to(self.dtype)   # weight_ph is float32
        cr = torch.clamp(r, -1.0, 1.0) if c["reward_clipping"] == "abs_one" else r         # :38-41
        discounts = (~d).to(self.dtype) * c["discount_factor"]                            # :43
        main_q, taps = dueling_network(self.params, x, pa, A, return_taps=True)           # model/apex_value.py:45-50
        with torch.no_grad():                                                              # no gradient reaches these
            saved = it._PATTERN["masks"]
            it._PATTERN["masks"] = None          # the ReLU pattern override only applies to the differentiated pass
            try:
                next_main_q = dueling_network(self.params, nx, a, A)                      # :52-57
                target_q = dueling_network(self.target, nx, a, A)                         # :59-64
            finally:
                it._PATTERN["masks"] = saved
        if next_action is None:
            next_action = torch.argmax(next_main_q, dim=1)                                 # :56 (first maximal index)
        else:
            next_action = torch.from_numpy(np.asarray(next_action).astype(np.int64))
        sav = take_state_action_value(main_q, a, A)                                        # :57-58
        nsav = take_state_action_value(target_q, next_action, A)                           # :59-60
        target_value = (nsav * discounts + cr).detach()                                    # :61
        td_error = (target_value - sav) ** 2                                               # :63
        value_loss = torch.mean(td_error * w)                                              # :64-65
        return dict(main_q=main_q, next_main_q=next_main_q, target_q=target_q, next_action=next_action,
                    state_action_value=sav, target_value=target_value, value_loss=value_loss, taps=taps)

    def get_td_error(self, state, next_state, previous_action, action, reward, done):
        """agent/apex.py:116-133 -> |target_value - state_action_value| [n]."""
        with torch.no_grad():
            o = self.losses(state, next_state, previous_action, action, reward, done)
        return np.abs(o["target_value"].numpy() - o["state_action_value"].numpy())

    def gradients(self, *batch, **kw):
        out = self.losses(*batch, **kw)
        names = list(self.params)
        extra = [k for k in ("a1", "a2", "a3") if k in out["taps"]]
        grads = torch.autograd.grad(out["value_loss"], [self.params[n] for n in names] +
                                    [out["taps"][k] for k in extra], allow_unused=True)
        g = OrderedDict((n, (gi if gi is not None else torch.zeros_like(self.params[n])))
                        for n, gi in zip(names, grads))
        out["act_grads"] = {k: gi for k, gi in zip(extra, grads[len(names):])}
        return out, g

    def distributed_train(self, state, next_state, previous_action, action, reward, done, is_weight,
                          return_all=False, next_action=None):
        """agent/apex.py:135-154 -> (loss, |target_value - state_action_value|), values from BEFORE the update."""
        c = self.cfg
        out, g = self.gradients(state, next_state, previous_action, action, reward, done, is_weight=is_weight,
                                next_action=next_action)
        lr = it.polynomial_decay_f32(c["start_learning_rate"], self.step, c["learning_frame"],
                                     c["end_learning_rate"])                                # :71
        # tf.clip_by_global_norm over the main variables (the target variables have gradient None and are skipped)
        gn = it.global_norm(g.values(), self.dtype)
        scale = it.clip_scale(gn, c["gradient_clip_norm"])
        # ApplyAdam (TF 1.14 training_ops): alpha = lr * sqrt(1 - beta2_power) / (1 - beta1_power);
        # m += (g - m)(1 - beta1); v += (g^2 - v)(1 - beta2); var -= m * alpha / (sqrt(v) + eps)
        b1p, b2p = float(self.beta1_power), float(self.beta2_power)
        alpha = float(lr) * np.sqrt(1.0 - b2p) / (1.0 - b1p)
        with torch.no_grad():
            for n, p in self.params.items():
                gc = g[n] * scale
                self.m[n] += (gc - self.m[n]) * (1.0 - BETA1)
                self.v[n] += (gc * gc - self.v[n]) * (1.0 - BETA2)
                p -= self.m[n] * alpha / (torch.sqrt(self.v[n]) + ADAM_EPS)
        self.beta1_power = np.float32(self.beta1_power * np.float32(BETA1))
        self.beta2_power = np.float32(self.beta2_power * np.float32(BETA2))
        self.step += 1
        td = np.abs(out["target_value"].numpy() - out["state_action_value"].detach().numpy())
        res = (float(out["value_loss"].detach().item()), td)
        if return_all:
            return res, out, g, float(gn), float(lr)
        return res

    def train(self, state, next_state, previous_action, action, reward, done):
        """agent/apex.py:156-168: the same update with unit importance weights."""
        return self.distributed_train(state, next_state, previous_action, action, reward, done,
                                      np.ones_like(np.asarray(reward, dtype=np.float32)))[0]


def make_transitions(B, A=4, input_shape=(84, 84, 4), seed=4321):
    """Seeded synthetic Ape-X minibatch: the field order and dtypes of train_apex.py:127-141
    (state, next_state uint8 [B,84,84,4]; previous_action, action int32; reward float32; done bool; is_weight)."""
    rng = np.random.default_rng(seed)
    state = rng.integers(0, 256, (B, *input_shape), dtype=np.uint8)
    next_state = rng.integers(0, 256, (B, *input_shape), dtype=np.uint8)
    previous_action = rng.integers(0, A, (B,)).astype(np.int32)
    action = rng.integers(0, A, (B,)).astype(np.int32)
    reward = rng.standard_normal((B,)).astype(np.float32)
    reward[rng.random(B) < 0.2] = 0.0
    big = rng.random(B) < 0.1
    reward[big] = (reward[big] * 4.0).astype(np.float32)
    done = rng.random(B) < 0.1
    is_weight = rng.uniform(0.2, 1.0, (B,)).astype(np.float32)
    is_weight[rng.integers(0, B)] = 1.0                       # Memory.sample normalises by the maximum
    return dict(state=state, next_state=next_state, previous_action=previous_action, action=action,
                reward=reward, done=done, is_weight=is_weight)


TRAIN_FIELDS = ("state", "next_state", "previous_action", "action", "reward", "done", "is_weight")
