"""H100-native stand-in for the reference's ``model/r2d2_lstm.py``: parameter inventory / initialisation of one scope
('main' or 'target') in TF layouts and TF variable-creation order (conv2d x3, dense x2 (action embedding),
rnn/lstm_cell kernel [3136 + 256 + L, 4L] gate order i,j,f,o + bias, dense 128, dense A (value), dense 1 (mean)).
The graph itself (``network`` :28-53, ``build_network`` :55-116) is evaluated by ``drl_r2d2_*`` through
``agent/r2d2.py`` (``Agent.get_action`` = one ``network`` step, ``Agent.train`` / ``main_q_value_test`` = the unroll)."""
import math

import numpy as np


def param_specs(num_action=4, lstm_size=64, input_shape=(84, 84, 1)):
    h, w, c = input_shape
    o1 = ((h - 8) // 4 + 1, (w - 8) // 4 + 1)
    o2 = ((o1[0] - 4) // 2 + 1, (o1[1] - 4) // 2 + 1)
    o3 = (o2[0] - 2, o2[1] - 2)
    cat, L = o3[0] * o3[1] * 64 + 256, lstm_size
    return [("conv1.w", (8, 8, c, 32)), ("conv1.b", (32,)), ("conv2.w", (4, 4, 32, 64)), ("conv2.b", (64,)),
            ("conv3.w", (3, 3, 64, 64)), ("conv3.b", (64,)), ("emb1.w", (num_action, 256)), ("emb1.b", (256,)),
            ("emb2.w", (256, 256)), ("emb2.b", (256,)), ("lstm.w", (cat + L, 4 * L)), ("lstm.b", (4 * L,)),
            ("q1.w", (L, 128)), ("q1.b", (128,)), ("value.w", (128, num_action)), ("value.b", (num_action,)),
            ("mean.w", (128, 1)), ("mean.b", (1,))]


def param_count(**kw):
    return sum(int(np.prod(s)) for _, s in param_specs(**kw))


def init_params(seed=None, **kw):
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
