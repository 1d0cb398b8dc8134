"""H100-native stand-in for the reference's ``model/impala_actor_critic.py``.

The reference builds a TF1 graph: conv 8x8s4/32 -> 4x4s2/64 -> 3x3s1/64 -> flatten(3136) ||
one_hot(prev_action) -> dense256 -> dense256 || one LSTMCell(256) step from FED (h, c) ->
actor [256,256,A+softmax] and critic [256,256,1] heads (model/impala_actor_critic.py:5-42), unrolled
as 3 x (T-2) per-timestep copies (:44-118).  Here the same functions evaluate eagerly on the GPU
through the C-ABI learner (``drl_learner_act`` / ``drl_learner_forward``); the variables live in a
module-level store that plays the role of ``tf.variable_scope('impala', reuse=tf.AUTO_REUSE)``.

Parameter inventory and TF layouts (conv HWIO, dense [in,out], LSTM [in+h, 4*units] with gate
order i,j,f,o; forget_bias 1.0 is NOT in the bias) -- TF1 variable-creation order:
conv2d, conv2d_1, conv2d_2, dense, dense_1, rnn/lstm_cell, dense_2..4 (actor), dense_5..7 (critic).
"""
import math

import numpy as np

from ..learner import NativeLearner


def param_specs(num_action=18, lstm_hidden_size=256, input_shape=(84, 84, 4)):
    """[(name, shape)] in flat-vector order; 4,153,267 floats for the reference geometry."""
    h, w, c = input_shape
    o1 = ((h - 8) // 4 + 1, (w - 8) // 4 + 1)
    o2 = ((o1[0] - 4) // 2 + 1, (o1[1] - 4) // 2 + 1)
    o3 = (o2[0] - 2, o2[1] - 2)
    flat, L = o3[0] * o3[1] * 64, lstm_hidden_size
    return [("conv1.w", (8, 8, c, 32)), ("conv1.b", (32,)), ("conv2.w", (4, 4, 32, 64)), ("conv2.b", (64,)),
            ("conv3.w", (3, 3, 64, 64)), ("conv3.b", (64,)), ("emb1.w", (num_action, 256)), ("emb1.b", (256,)),
            ("emb2.w", (256, 256)), ("emb2.b", (256,)), ("lstm.w", (flat + 256 + L, 4 * L)), ("lstm.b", (4 * L,)),
            ("actor1.w", (L, 256)), ("actor1.b", (256,)), ("actor2.w", (256, 256)), ("actor2.b", (256,)),
            ("actor3.w", (256, num_action)), ("actor3.b", (num_action,)),
            ("critic1.w", (L, 256)), ("critic1.b", (256,)), ("critic2.w", (256, 256)), ("critic2.b", (256,)),
            ("critic3.w", (256, 1)), ("critic3.b", (1,))]


def param_count(**kw):
    return sum(int(np.prod(s)) for _, s in param_specs(**kw))


def init_params(seed=None, **kw):
    """TF defaults: glorot-uniform kernels U(+-sqrt(6/(fan_in+fan_out))), zero biases.  Returns the flat
    float32 vector (what ``global_variables_initializer`` would produce, agent/impala.py:114-116)."""
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


def split_flat(flat, **kw):
    """flat vector -> {name: ndarray view in TF layout}."""
    out, off = {}, 0
    for name, shape in param_specs(**kw):
        n = int(np.prod(shape))
        out[name] = flat[off:off + n].reshape(shape)
        off += n
    if off != flat.size:
        raise ValueError("flat vector has %d floats, expected %d" % (flat.size, off))
    return out


# ---- variable store ("impala" scope with AUTO_REUSE) -------------------------------------
_STORE = {"flat": None, "engine": None, "key": None}


def set_variables(flat):
    _STORE["flat"] = np.ascontiguousarray(flat, np.float32)
    if _STORE["engine"] is not None:
        _STORE["engine"].set_params(_STORE["flat"])


def get_variables():
    return _STORE["flat"]


def _engine(rows, num_action, lstm_hidden_size):
    """Forward-only engine with room for `rows` independent single-step rows (act() needs n <= B*T)."""
    key = (num_action, lstm_hidden_size)
    eng = _STORE["engine"]
    if eng is None or _STORE["key"] != key or eng.B * eng.T < rows:
        if eng is not None:
            eng.close()
        eng = NativeLearner(batch=max((rows + 2) // 3, 1), trajectory=3, num_action=num_action,
                            lstm_hidden_size=lstm_hidden_size, num_slots=1)
        if _STORE["flat"] is None:
            _STORE["flat"] = init_params(num_action=num_action, lstm_hidden_size=lstm_hidden_size)
        eng.set_params(_STORE["flat"])
        _STORE["engine"], _STORE["key"] = eng, key
    return eng


def _to_u8(image):
    a = np.asarray(image)
    if a.dtype == np.uint8:
        return a
    # the reference feeds state/255 as float32 (agent/impala.py:133); the kernels take the raw bytes
    return np.clip(np.rint(a * 255.0), 0, 255).astype(np.uint8)


def network(image, previous_action, initial_h, initial_c, num_action, lstm_hidden_size):
    """model/impala_actor_critic.py:33-42 -> (actor softmax [N,A], critic [N], c [N,L], h [N,L])."""
    img = _to_u8(image)
    n = img.shape[0]
    eng = _engine(n, num_action, lstm_hidden_size)
    pol, h, c = eng.act(img, previous_action, initial_h, initial_c)
    # value is produced by the same forward; read it back from the activation buffer (time-major == row order here)
    val = eng.read_buffer("value", eng.B * eng.T)[:n].copy()
    return pol, val, c, h


def build_network(state, previous_action, initial_h, initial_c,
                  trajectory_state, trajectory_previous_action,
                  trajectory_initial_h, trajectory_initial_c,
                  num_action, lstm_hidden_size, trajectory):
    """model/impala_actor_critic.py:44-118 -> (policy, c, h, first_policy, first_value, middle_policy,
    middle_value, last_policy, last_value).  The three windows are slices of ONE forward over the T
    distinct rows (the reference evaluates 3 x (T-2) overlapping copies of the same function)."""
    policy, _, c, h = network(state, previous_action, initial_h, initial_c, num_action, lstm_hidden_size)
    ts = _to_u8(trajectory_state)
    B, T = ts.shape[0], ts.shape[1]
    if T != trajectory:
        raise ValueError("trajectory_state has T=%d, expected %d" % (T, trajectory))
    pol = np.empty((B, T, num_action), np.float32)
    val = np.empty((B, T), np.float32)
    tpa = np.asarray(trajectory_previous_action)
    th = np.asarray(trajectory_initial_h, np.float32)
    tc = np.asarray(trajectory_initial_c, np.float32)
    for t in range(T):      # T batched forwards of B rows each
        p, v, _, _ = network(ts[:, t], tpa[:, t], th[:, t], tc[:, t], num_action, lstm_hidden_size)
        pol[:, t], val[:, t] = p, v
    return (policy, c, h, pol[:, :-2], val[:, :-2], pol[:, 1:-1], val[:, 1:-1], pol[:, 2:], val[:, 2:])
