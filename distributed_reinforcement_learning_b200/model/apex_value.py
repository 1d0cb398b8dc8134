"""H100-native stand-in for the reference's ``model/apex_value.py`` (the Ape-X dueling network).

Reference graph (model/apex_value.py:4-41): conv 8x8s4/32 -> 4x4s2/64 -> 3x3s1/64 -> flatten(3136) ||
one_hot(previous_action) -> dense256 -> dense256; concat (3392) -> value stream [256, 256, A] and a SEPARATE
"mean" stream [256, 256, 1]; q = value - mean (the subtraction broadcasts the scalar stream; it is not the
mean of the advantages).  ``build_network`` (:43-66) evaluates main(s, prev_a), main(s', a) and target(s', a).
Here the same functions evaluate eagerly on the GPU through ``drl_apex_*``; the variables of the two scopes live
in a module-level store.

Parameter inventory per scope, TF1 variable-creation order: conv2d, conv2d_1, conv2d_2, dense, dense_1 (embedding),
dense_2..4 (value stream), dense_5..7 (mean stream); conv HWIO, dense [in, out].
"""
import math

import numpy as np

from ..apex_learner import MAIN, TARGET, NativeApexLearner


def param_specs(num_action=4, input_shape=(84, 84, 4), hidden_list=(256, 256)):
    if tuple(hidden_list) != (256, 256):
        raise ValueError("only hidden_list=[256, 256] (agent/apex.py:51) is supported")
    h, w, c = input_shape
    o1 = ((h - 8) // 4 + 1, (w - 8) // 4 + 1)
    o2 = ((o1[0] - 4) // 2 + 1, (o1[1] - 4) // 2 + 1)
    o3 = (o2[0] - 2, o2[1] - 2)
    cat = o3[0] * o3[1] * 64 + 256
    return [("conv1.w", (8, 8, c, 32)), ("conv1.b", (32,)), ("conv2.w", (4, 4, 32, 64)), ("conv2.b", (64,)),
            ("conv3.w", (3, 3, 64, 64)), ("conv3.b", (64,)), ("emb1.w", (num_action, 256)), ("emb1.b", (256,)),
            ("emb2.w", (256, 256)), ("emb2.b", (256,)),
            ("value1.w", (cat, 256)), ("value1.b", (256,)), ("value2.w", (256, 256)), ("value2.b", (256,)),
            ("value3.w", (256, num_action)), ("value3.b", (num_action,)),
            ("mean1.w", (cat, 256)), ("mean1.b", (256,)), ("mean2.w", (256, 256)), ("mean2.b", (256,)),
            ("mean3.w", (256, 1)), ("mean3.b", (1,))]


def param_count(**kw):
    return sum(int(np.prod(s)) for _, s in param_specs(**kw))


def init_params(seed=None, **kw):
    """TF defaults (glorot-uniform kernels, zero biases) as one flat float32 vector of ONE scope."""
    rng = np.random.default_rng(seed)
    parts = []
    for name, shape in param_specs(**kw):
        if name.endswith(".b"):
            parts.append(np.zeros(shape, np.float32).ravel())
            continue
        if len(shape) == 4:
            rf = shape[0] * shape[1]
            fan_in, fan_out = rf * shape[2], rf * shape[3]
        else:
            fan_in, fan_out = shape
        lim = math.sqrt(6.0 / (fan_in + fan_out))
        parts.append(rng.uniform(-lim, lim, size=shape).astype(np.float32).ravel())
    return np.concatenate(parts)


# ---- variable store (scopes 'main' and 'target') ---------------------------------------
_STORE = {"main": None, "target": None, "engine": None, "key": None}


def set_variables(main=None, target=None):
    for k, v in (("main", main), ("target", target)):
        if v is not None:
            _STORE[k] = np.ascontiguousarray(v, np.float32)
            if _STORE["engine"] is not None:
                _STORE["engine"].set_params(_STORE[k], MAIN if k == "main" else TARGET)


def _engine(rows, num_action):
    eng = _STORE["engine"]
    if eng is None or _STORE["key"] != num_action or 2 * eng.B < rows:
        if eng is not None:
            eng.close()
        eng = NativeApexLearner(batch=max((rows + 1) // 2, 1), num_action=num_action, num_slots=1)
        for k, which, seed in (("main", MAIN, None), ("target", TARGET, None)):
            if _STORE[k] is None:
                _STORE[k] = init_params(seed, num_action=num_action)
            eng.set_params(_STORE[k], which)
        _STORE["engine"], _STORE["key"] = eng, num_action
    return eng


def _to_u8(image):
    a = np.asarray(image)
    if a.dtype == np.uint8:
        return a
    return np.clip(np.rint(a * 255.0), 0, 255).astype(np.uint8)     # the reference feeds state / 255


def dueling_network(image, previous_action, num_action, hidden_list, scope="main"):
    """model/apex_value.py:22-41 -> q_value [N, A] of scope 'main' (the 'target' scope is evaluated by
    ``build_network``)."""
    if scope != "main":
        raise ValueError("dueling_network evaluates the 'main' scope; use build_network for 'target'")
    param_specs(num_action, hidden_list=hidden_list)
    img = _to_u8(image)
    return _engine(img.shape[0], num_action).act(img, previous_action)


def build_network(current_state, next_state, previous_action, action, num_action, hidden_list):
    """model/apex_value.py:43-66 -> (main_q_value, next_main_q_value, target_q_value), each [N, A]."""
    param_specs(num_action, hidden_list=hidden_list)
    s, ns = _to_u8(current_state), _to_u8(next_state)
    n = s.shape[0]
    eng = _engine(2 * n, num_action)
    zeros = np.zeros(n, np.float32)
    eng.td_error(s, ns, previous_action, action, zeros, np.zeros(n, np.uint8))
    t = eng.taps(n)
    return t["main_q"], t["next_main_q"], t["target_q"]
