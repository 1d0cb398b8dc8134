"""H100-native stand-in for the reference's ``optimizer/vtrace.py`` (same names, argument order,
layouts and error behaviour; NumPy arrays in and out, CUDA kernels underneath via the C-ABI).

  split_data                          optimizer/vtrace.py:3-14   (views, no compute)
  log_probs_from_softmax_and_actions  optimizer/vtrace.py:16-27
  from_softmax                        optimizer/vtrace.py:29-69   -> drl_vtrace_from_softmax
  from_importance_weights             optimizer/vtrace.py:71-103  -> drl_vtrace_from_importance_weights
  compute_policy_gradient_loss        optimizer/vtrace.py:105-112
  compute_baseline_loss               optimizer/vtrace.py:114-118
  compute_entropy_loss                optimizer/vtrace.py:120-126

In the learner these are not called one by one: ``agent/impala.py`` runs the fused
V-trace + loss + head-gradient kernel (csrc/vtrace.cu).  The stand-alone forms exist for parity
tests and for callers that used the reference functions directly.
"""
import numpy as np

from .. import _native as N


def split_data(x):
    """first / middle / last windows x[:, :-2], x[:, 1:-1], x[:, 2:] (optimizer/vtrace.py:3-14)."""
    return x[:, :-2], x[:, 1:-1], x[:, 2:]


def _clip_arg(clip_rho_threshold):
    return -1.0 if clip_rho_threshold is None else float(clip_rho_threshold)


def from_importance_weights(log_rhos, discounts, rewards, values, bootstrap_value,
                            clip_rho_threshold=1.0, clip_pg_rho_threshold=1.0):
    """Time-major [T, B] inputs, bootstrap_value [B] -> (vs, clipped_rhos) [T, B].
    ``clip_pg_rho_threshold`` is accepted and unused, as in the reference (optimizer/vtrace.py:72)."""
    lr = N.as_c(log_rhos, np.float32)
    if lr.ndim != 2:
        raise ValueError("log_rhos must be [T, B]")
    T, B = lr.shape
    g = N.as_c(discounts, np.float32, (T, B), "discounts")
    r = N.as_c(rewards, np.float32, (T, B), "rewards")
    v = N.as_c(values, np.float32, (T, B), "values")
    boot = N.as_c(bootstrap_value, np.float32, (B,), "bootstrap_value")
    vs = np.empty((T, B), np.float32)
    rho = np.empty((T, B), np.float32)
    N.check(N.lib.drl_vtrace_from_importance_weights(N.ptr(lr), N.ptr(g), N.ptr(r), N.ptr(v), N.ptr(boot), T, B,
                                                     _clip_arg(clip_rho_threshold), N.ptr(vs), N.ptr(rho)))
    return vs, rho


def from_softmax(behavior_policy_softmax, target_policy_softmax, actions, discounts,
                 rewards, values, next_values, action_size, clip_rho_threshold=1.0,
                 clip_pg_rho_threshold=1.0):
    """Batch-major [B, T, A] / [B, T] inputs -> (vs, clipped_rho) [B, T] (optimizer/vtrace.py:29-69)."""
    mu = N.as_c(behavior_policy_softmax, np.float32)
    if mu.ndim != 3 or mu.shape[2] != action_size:
        raise ValueError("behavior_policy_softmax must be [B, T, %d]" % action_size)
    B, T, A = mu.shape
    pi = N.as_c(target_policy_softmax, np.float32, (B, T, A), "target_policy_softmax")
    a = N.as_c(actions, np.int32, (B, T), "actions")
    g = N.as_c(discounts, np.float32, (B, T), "discounts")
    r = N.as_c(rewards, np.float32, (B, T), "rewards")
    v = N.as_c(values, np.float32, (B, T), "values")
    nv = N.as_c(next_values, np.float32, (B, T), "next_values")
    vs = np.empty((B, T), np.float32)
    rho = np.empty((B, T), np.float32)
    N.check(N.lib.drl_vtrace_from_softmax(N.ptr(mu), N.ptr(pi), N.ptr(a), N.ptr(g), N.ptr(r), N.ptr(v), N.ptr(nv),
                                          B, T, A, _clip_arg(clip_rho_threshold), N.ptr(vs), N.ptr(rho)))
    return vs, rho


def _losses(softmax, actions, advantages, vs, value):
    sm = N.as_c(softmax, np.float32)
    if sm.ndim != 3:
        raise ValueError("softmax must be [B, T, A]")
    B, T, A = sm.shape
    a = N.as_c(actions if actions is not None else np.zeros((B, T), np.int32), np.int32, (B, T), "actions")
    adv = N.as_c(advantages if advantages is not None else np.zeros((B, T), np.float32), np.float32, (B, T),
                 "advantages")
    vs_ = N.as_c(vs if vs is not None else np.zeros((B, T), np.float32), np.float32, (B, T), "vs")
    val = N.as_c(value if value is not None else np.zeros((B, T), np.float32), np.float32, (B, T), "value")
    sums = np.zeros(3, np.float32)
    logp = np.empty((B, T), np.float32)
    N.check(N.lib.drl_vtrace_loss_sums(N.ptr(sm), N.ptr(a), N.ptr(adv), N.ptr(vs_), N.ptr(val), B, T, A,
                                       N.ptr(sums), N.ptr(logp)))
    return sums, logp


def log_probs_from_softmax_and_actions(policy_softmax, actions, action_size):
    """log(sum_a p * onehot(a)), no epsilon (optimizer/vtrace.py:16-27)."""
    sm = np.asarray(policy_softmax)
    if sm.shape[-1] != action_size:
        raise ValueError("policy_softmax last dim must be action_size")
    return _losses(sm, actions, None, None, None)[1]


def compute_policy_gradient_loss(softmax, actions, advantages, output_size):
    """-sum log(pi(a) + 1e-8) * advantages (optimizer/vtrace.py:105-112)."""
    return float(_losses(softmax, actions, advantages, None, None)[0][0])


def compute_baseline_loss(vs, value):
    """0.5 * sum (vs - value)^2 (optimizer/vtrace.py:114-118)."""
    v = np.asarray(value, np.float32)
    dummy = np.full(v.shape + (1,), 1.0, np.float32)
    return float(_losses(dummy, None, None, vs, v)[0][1])


def compute_entropy_loss(softmax):
    """sum pi * log(pi) (= -entropy, no epsilon) (optimizer/vtrace.py:120-126)."""
    return float(_losses(softmax, None, None, None, None)[0][2])
