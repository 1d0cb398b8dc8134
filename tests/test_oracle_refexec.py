"""PIN of the oracle to the reference itself: the UNMODIFIED reference files (``/root/reference/agent/impala.py``,
``optimizer/vtrace.py``, ``model/impala_actor_critic.py``, ``distributed_queue/buffer_queue.py``, ``utils.py``; and the
Ape-X / R2D2 files) are imported and executed here over ``oracle/tf1_shim`` (a TF 1.14 API stand-in on torch-CPU that
restates only TF's op semantics -- see its docstring) and must agree with the restatements under ``oracle/`` on every
slice, window, loss, stop_gradient and optimizer decision: V-trace taps, the three losses, all 24 gradients, three
RMSProp steps with slots and global_step, both reward-clipping modes, the reference-shaped 54-copy graph against the
deduplicated forward, variable names/order/sharing, parameter_sync, single-step inference and the FIFO queue's order.

CPU-only.  Where the reference checkout is present (``oracle/ref_exec.py``) its files are executed; everywhere else
the results of those executions are read from ``tests/golden/refexec/<test>.npz``, written by the same code with
``DRL_WRITE_REFEXEC_GOLDEN=1`` (tensors larger than 2048 elements are stored as a fixed, seeded sample of 256 entries
plus their absolute maximum, the denominator of the relative error).  The restatements are compared either way."""
import os

import numpy as np
import pytest
import torch

from oracle import impala_torch as it
from oracle import ref_exec, synthetic, vtrace_np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refexec")
_BIG, _SAMPLE = 2048, 256


def _sample_idx(size):
    return np.sort(np.random.default_rng(0).choice(size, _SAMPLE, replace=False))


class Sampled:
    """A stored sample of a large reference tensor: values at the seeded flat indices _sample_idx(size), max |x| over
    the whole tensor."""

    def __init__(self, val, absmax, shape):
        self.shape, self.val, self.absmax = tuple(int(x) for x in shape), val, float(absmax)
        self.idx = _sample_idx(int(np.prod(self.shape)))


def _pack(d):
    out = {}
    for k, v in d.items():
        a = np.asarray(v)
        if a.dtype.kind in "fiu" and a.size > _BIG:
            out[k + "__val"], out[k + "__absmax"] = a.ravel()[_sample_idx(a.size)], np.abs(a).max()
            out[k + "__shape"] = np.array(a.shape, np.int64)
        else:
            out[k] = a
    return out


def _unpack(z):
    d = {}
    for k in z.files:
        if k.endswith("__shape"):
            b = k[:-7]
            d[b] = Sampled(z[b + "__val"], z[b + "__absmax"], z[k])
        elif not k.endswith(("__val", "__absmax")):
            d[k] = z[k]
    return d


def reference(name, compute):
    """What the executed reference returns for test `name`: computed when the checkout is present (and stored with
    DRL_WRITE_REFEXEC_GOLDEN=1), else the stored copy."""
    path = os.path.join(GOLDEN, name + ".npz")
    if ref_exec.available():
        d = compute()
        if os.environ.get("DRL_WRITE_REFEXEC_GOLDEN") == "1":
            os.makedirs(GOLDEN, exist_ok=True)
            np.savez_compressed(path, **_pack(d))
        return d
    with np.load(path) as z:
        return _unpack(z)


def sub(d, prefix):
    """The entries of d under `prefix/`, keyed by the rest of the name."""
    return {k[len(prefix) + 1:]: v for k, v in d.items() if k.startswith(prefix + "/")}


F64 = dict(rtol=0, atol=0)


def _rel(a, b):
    if isinstance(b, Sampled):
        a = np.asarray(a, np.float64).reshape(-1)
        assert a.size == int(np.prod(b.shape)), (a.size, b.shape)
        return float(np.max(np.abs(a[b.idx] - b.val.astype(np.float64))) / max(b.absmax, 1e-300))
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)) if b.size else 0.0


def _case(B, T, A, seed=4321, **cfg):
    batch = synthetic.make_batch(B, T=T, A=A, seed=seed)
    params = it.init_params(0, torch.float32, num_action=A)
    return batch, params, [batch[k] for k in synthetic.TRAIN_FIELDS], dict(trajectory=T, num_action=A, **cfg)


TAPS = ("vs", "clipped_rho", "vs_plus_1", "pg_advantage", "pi_loss", "baseline_loss", "entropy", "total_loss")


@pytest.mark.parametrize("clipping", ["abs_one", "soft_asymmetric"])
def test_impala_executed_reference_equals_restatement(clipping):
    """agent/impala.py:31-100,132-148 executed == oracle/impala_torch.py (reference-shaped AND deduplicated)."""
    batch, params, args, cfg = _case(2, 6, 18, reward_clipping=clipping)
    names = TAPS + ("unrolled_first_policy", "unrolled_first_value", "unrolled_middle_value", "unrolled_last_value",
                    "discounts", "clipped_r_ph")

    def compute():
        R = ref_exec.ReferenceImpala(params, **cfg)
        f = R.fetch(args, names)
        d = {"f/" + k: f[k] for k in names}
        d.update({"g/" + n: v for n, v in R.gradients(args).items()})
        return d

    d = reference("impala_%s" % clipping, compute)
    f, rg = sub(d, "f"), sub(d, "g")
    for shaped, tol in (("reference", 1e-13), ("dedup", 1e-11)):
        L = it.Learner(params, torch.float64, shaped, **cfg)
        out, g = L.gradients(*args)
        for k in TAPS:
            assert _rel(out[k].detach().numpy(), f[k]) <= tol, (shaped, k)
        assert _rel(out["first_policy"].detach().numpy(), f["unrolled_first_policy"]) <= tol
        assert _rel(out["middle_value"].detach().numpy(), f["unrolled_middle_value"]) <= tol
        assert _rel(out["last_value"].detach().numpy(), f["unrolled_last_value"]) <= tol
        assert set(g) == set(rg) and len(rg) == 24
        for n in g:
            assert _rel(g[n].numpy(), rg[n]) <= tol * 10, (shaped, n)
    assert np.min(f["clipped_r_ph"]) >= (-1.0 if clipping == "abs_one" else -1.5)


def test_impala_three_train_steps_track_the_executed_reference():
    """Agent.train x3: returned scalars, every parameter, the RMSProp ``rms`` slots (ms0 = 1, eps inside the sqrt),
    global_step and the learning rate -- TF1 optimizer semantics as restated in the shim's docstring."""
    batch, params, args, cfg = _case(2, 6, 18)

    def compute():
        R = ref_exec.ReferenceImpala(params, **cfg)
        d = {}
        for step in range(3):
            d["r%d" % step] = np.array(R.train(*args)[:4], np.float64)
            d["global_step%d" % step] = np.array(R.global_step())
            d.update({"p%d/%s" % (step, n): v for n, v in R.params().items()})
            d.update({"rms%d/%s" % (step, n): v for n, v in R.rms().items()})
        d["rms_moved_from_ones"] = np.array(all(np.any(v != 1.0) and np.all(v > 0.9) for v in R.rms().values()))
        return d

    d = reference("impala_three_steps", compute)
    L = it.Learner(params, torch.float64, "dedup", **cfg)
    for step in range(3):
        r, o = d["r%d" % step], L.train(*args)
        for a, b in zip(r[:3], o[:3]):
            assert abs(a - b) <= 1e-9 * max(abs(b), 1.0)
        assert abs(r[3] - o[3]) < 1e-10                  # lr: float32 polynomial_decay in the oracle, exact here
        assert int(d["global_step%d" % step]) == step + 1 == L.step
        for n, v in sub(d, "p%d" % step).items():
            assert _rel(L.params[n].detach().numpy(), v) < 1e-9, n
        for n, v in sub(d, "rms%d" % step).items():
            assert _rel(L.ms[n].numpy(), v) < 1e-9, n
    assert bool(d["rms_moved_from_ones"])                # slots started at ones (TF1), not zeros


def test_baseline_config0_b4_t20_54_graph_copies_equal_one_forward():
    """BASELINE configs[0] (T=20, B=4): the reference's 3 x 18 per-timestep network copies (executed) against the
    ONE forward over the 20 distinct rows that the CUDA path runs (shift identity, SURVEY App. C.4)."""
    batch, params, args, cfg = _case(4, 20, 18, seed=1234)

    def compute():
        R = ref_exec.ReferenceImpala(params, **cfg)
        f = R.fetch(args, TAPS)
        d = {"f/" + k: f[k] for k in TAPS}
        d.update({"g/" + n: v for n, v in R.gradients(args).items()})
        return d

    d = reference("impala_b4_t20", compute)
    f, rg = sub(d, "f"), sub(d, "g")
    L = it.Learner(params, torch.float64, "dedup", **cfg)
    out, g = L.gradients(*args)
    for k in TAPS:
        assert _rel(out[k].detach().numpy(), f[k]) <= 1e-11, k
    for n in g:
        assert _rel(g[n].numpy(), rg[n]) <= 1e-10, n


def test_float32_execution_is_within_the_parity_bar_of_float64():
    """The same reference graph evaluated in float32 (TF's arithmetic type) sits inside the 1e-4 bar that the CUDA path
    is held to: the bar is meaningful for a float32 implementation of this graph."""
    batch, params, args, cfg = _case(2, 6, 18)

    def compute():
        f64 = ref_exec.ReferenceImpala(params, **cfg).fetch(args, TAPS)
        R32 = ref_exec.ReferenceImpala(params, float_dtype=torch.float32, **cfg)
        f32 = R32.fetch(args, TAPS)
        R32.ref.tf._shim.FLOAT = torch.float64
        d = {"f64/" + k: f64[k] for k in TAPS}
        d.update({"f32/" + k: f32[k] for k in TAPS})
        return d

    d = reference("impala_float32", compute)
    f64, f32 = sub(d, "f64"), sub(d, "f32")
    assert f32["vs"].dtype == np.float32
    L = it.Learner(params, torch.float64, "dedup", **cfg)
    out, _ = L.gradients(*args)
    for k in TAPS:
        assert _rel(f32[k], f64[k]) < 1e-4, k
        assert _rel(out[k].detach().numpy(), f64[k]) <= 1e-11, k


def test_variable_names_sharing_and_parameter_sync():
    """model/impala_actor_critic.py:47-109 re-enters variable_scope('impala', reuse=AUTO_REUSE) 55 times: exactly 24
    trainable variables result, named as TF1 names them; a second agent (train_impala.py:64-80, 'actor_0') adds its own
    24 and utils.copy_src_to_dst (parameter_sync) copies learner -> actor in creation order.  The single-step inference
    of the synced actor is compared with the oracle's ``network`` where the checkout is present (the 16 MB of synced
    parameters are not stored); the stored run keeps its policy / state invariants."""
    rng = np.random.default_rng(3)
    state = rng.integers(0, 256, (84, 84, 4), dtype=np.uint8)
    h, c = rng.standard_normal(256).astype(np.float32) * 0.3, rng.standard_normal(256).astype(np.float32)

    def compute():
        ref = ref_exec.load(float_dtype=torch.float64)
        tf = ref.tf
        kw = dict(trajectory=5, input_shape=[84, 84, 4], num_action=6, lstm_hidden_size=256, discount_factor=0.99,
                  start_learning_rate=6e-4, end_learning_rate=0.0, learning_frame=10 ** 9, baseline_loss_coef=1.0,
                  entropy_coef=0.05, gradient_clip_norm=40.0, reward_clipping="abs_one")
        learner = ref["agent.impala"].Agent(model_name="learner", learner_name="learner", **kw)
        d = {"names": np.array([v.op_name for v in tf.trainable_variables()]),
             "lstm_kernel_shape": np.array(tf.get_default_graph().var_by_name["learner/impala/rnn/lstm_cell/kernel"]._shape)}
        actor = ref["agent.impala"].Agent(model_name="actor_0", learner_name="learner", **kw)
        d["n_trainable_two_agents"] = np.array(len(tf.trainable_variables()))
        d["n_global_to_session"] = np.array(len(actor.global_to_session))
        sess = tf.Session()
        learner.set_session(sess)
        src, dst = tf.trainable_variables("learner"), tf.trainable_variables("actor_0")
        d["differ_before_sync"] = np.array(any(np.any(a.numpy() != b.numpy()) for a, b in zip(src, dst)))
        actor.sess = sess
        actor.parameter_sync()
        d["equal_after_sync"] = np.array(all(np.array_equal(a.numpy(), b.numpy()) for a, b in zip(src, dst)))
        np.random.seed(0)
        action, policy, mx, h1, c1 = actor.get_policy_and_action(state, 2, h, c)
        d.update(action=np.array(action), policy=np.asarray(policy), mx=np.array(mx), h1=np.asarray(h1), c1=np.asarray(c1))
        # single-step inference (agent/impala.py:118-130) on the synced actor == the oracle's ``network``
        p = {n: torch.from_numpy(v.numpy()) for n, v in zip([s for s, _ in it.param_specs(num_action=6)], dst)}
        x = torch.from_numpy((state[None].astype(np.float64) / 255).astype(np.float32)).double()
        pol, val, oc, oh = it.network(p, x, torch.tensor([2]), torch.from_numpy(h[None]).double(),
                                      torch.from_numpy(c[None]).double(), 6, 256)
        assert _rel(policy, pol[0].numpy()) < 1e-12
        assert _rel(h1, oh[0].numpy()) < 1e-12 and _rel(c1, oc[0].numpy()) < 1e-12      # returns (.., h, c) in that order
        return d

    d = reference("variable_names_and_sync", compute)
    names = [str(n) for n in d["names"]]
    assert len(names) == 24
    assert names[:2] == ["learner/impala/conv2d/kernel", "learner/impala/conv2d/bias"]
    assert names[10:12] == ["learner/impala/rnn/lstm_cell/kernel", "learner/impala/rnn/lstm_cell/bias"]
    assert names[-2:] == ["learner/impala/dense_7/kernel", "learner/impala/dense_7/bias"]
    assert len(it.param_specs(num_action=6)) == len(names)
    assert tuple(d["lstm_kernel_shape"]) == (3648, 1024)
    assert int(d["n_trainable_two_agents"]) == 48 and int(d["n_global_to_session"]) == 24
    assert bool(d["differ_before_sync"]) and bool(d["equal_after_sync"])
    policy = d["policy"]
    assert policy.shape == (6,) and abs(float(policy.sum()) - 1.0) < 1e-6 and float(d["mx"]) == float(policy.max())
    assert 0 <= int(d["action"]) < 6 and d["h1"].shape == (256,) and d["c1"].shape == (256,)


def test_static_placeholder_shapes_reject_a_wrong_trajectory_length():
    """Error behaviour at the boundary (SURVEY 8b): feeding T+1 steps to the [None, T, ...] placeholders raises; the
    restatement rejects the same batch."""
    batch, params, args, cfg = _case(2, 6, 18)
    bad = synthetic.make_batch(2, T=7, A=18, seed=1)
    bad_args = [bad[k] for k in synthetic.TRAIN_FIELDS]

    def compute():
        R = ref_exec.ReferenceImpala(params, **cfg)
        try:
            R.train(*bad_args)
        except ValueError:
            return {"raised_value_error": np.array(True)}
        return {"raised_value_error": np.array(False)}

    d = reference("placeholder_shapes", compute)
    assert bool(d["raised_value_error"])
    L = it.Learner(params, torch.float64, "dedup", **cfg)
    with pytest.raises((ValueError, RuntimeError, AssertionError, IndexError)):
        L.train(*bad_args)


# ---- optimizer/vtrace.py, function by function -------------------------------------------------------------------
def _run(ref, tensors, feeds=None):
    return ref.tf.Session().run(tensors, feed_dict=feeds)


def test_vtrace_functions_executed_equal_numpy_and_c_restatements():
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "vtrace_T18_B8.npz"))
    kw = {k: z[k] for k in ("log_rhos", "discounts", "rewards", "values", "bootstrap_value")}
    rng = np.random.default_rng(11)
    B, T, A = 5, 9, 7
    sm = lambda x: np.exp(x) / np.exp(x).sum(-1, keepdims=True)
    mu, pi = sm(rng.standard_normal((B, T, A))), sm(rng.standard_normal((B, T, A)))
    act = rng.integers(0, A, (B, T)).astype(np.int32)
    disc = (rng.random((B, T)) > 0.1) * 0.99
    rew, val, nval = rng.standard_normal((B, T)), rng.standard_normal((B, T)), rng.standard_normal((B, T))
    adv = rng.standard_normal((B, T))

    def compute():
        ref = ref_exec.load(("optimizer.vtrace",), float_dtype=torch.float64)
        vt, tf = ref["optimizer.vtrace"], ref.tf
        c = tf.constant
        d = {}
        d["vs"], d["rho"] = _run(ref, list(vt.from_importance_weights(**{k: c(v) for k, v in kw.items()})))
        # clip_rho_threshold honoured, clip_pg_rho_threshold dead, cs hard-coded at 1 (optimizer/vtrace.py:72-80)
        d["vs_clip"], d["rho_clip"] = _run(ref, list(vt.from_importance_weights(
            clip_rho_threshold=0.5, clip_pg_rho_threshold=7.0, **{k: c(v) for k, v in kw.items()})))
        d["sm_vs"], d["sm_rho"] = _run(ref, list(vt.from_softmax(c(mu), c(pi), c(act), c(disc), c(rew), c(val), c(nval), A)))
        got = _run(ref, [vt.compute_policy_gradient_loss(c(pi), c(act), c(adv), A), vt.compute_baseline_loss(c(val), c(nval)),
                         vt.compute_entropy_loss(c(pi)), vt.log_probs_from_softmax_and_actions(c(pi), c(act), A)] +
                   list(vt.split_data(c(val))))
        d.update(pg_loss=np.array(got[0]), baseline_loss=np.array(got[1]), entropy_loss=np.array(got[2]), log_probs=got[3])
        d.update({"split%d" % i: g for i, g in enumerate(got[4:])})
        return d

    d = reference("vtrace_functions", compute)
    np.testing.assert_allclose(d["vs"], z["vs"], rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(d["rho"], z["clipped_rhos"], rtol=1e-13, atol=1e-13)
    ovs, orho = vtrace_np.from_importance_weights(**kw)
    np.testing.assert_allclose(d["vs"], ovs, rtol=1e-13, atol=1e-13)
    from oracle import vtrace_c
    cvs, crho = vtrace_c.from_importance_weights(**kw)               # plain-C restatement (gcc, built on demand)
    np.testing.assert_allclose(d["vs"], cvs, rtol=1e-12, atol=1e-12)
    b = vtrace_np.from_importance_weights(clip_rho_threshold=0.5, **kw)
    np.testing.assert_allclose(d["vs_clip"], b[0], rtol=1e-13, atol=1e-13)
    assert d["rho_clip"].max() <= 0.5
    exp = vtrace_np.from_softmax(mu, pi, act, disc, rew, val, nval, A)
    np.testing.assert_allclose(d["sm_vs"], exp[0], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(d["sm_rho"], exp[1], rtol=1e-12, atol=1e-12)
    assert float(d["pg_loss"]) == pytest.approx(vtrace_np.compute_policy_gradient_loss(pi, act, adv, A), rel=1e-12)
    assert float(d["baseline_loss"]) == pytest.approx(vtrace_np.compute_baseline_loss(val, nval), rel=1e-12)
    assert float(d["entropy_loss"]) == pytest.approx(vtrace_np.compute_entropy_loss(pi), rel=1e-12)
    np.testing.assert_allclose(d["log_probs"], vtrace_np.log_probs_from_softmax_and_actions(pi, act, A), rtol=1e-12)
    splits = vtrace_np.split_data(val)
    assert len([k for k in d if k.startswith("split")]) == len(splits)
    for i, e in enumerate(splits):
        np.testing.assert_array_equal(d["split%d" % i], e)


# ---- distributed_queue/buffer_queue.py:418-512 against the pinned-ring replacement ---------------------------------
FIFO_FIELDS = ("state", "next_state", "reward", "done", "behavior_policy", "action", "previous_action", "previous_h",
               "previous_c")


def test_reference_fifo_queue_order_equals_the_ring(native_or_none=None):
    T, shape, A, L, cap, batch = 5, [6, 6, 2], 4, 8, 8, 3
    rng = np.random.default_rng(5)

    def rec():
        return dict(unrolled_state=rng.integers(0, 256, (T, *shape), dtype=np.uint8),
                    unrolled_next_state=rng.integers(0, 256, (T, *shape), dtype=np.uint8),
                    unrolled_reward=rng.standard_normal(T).astype(np.float32), unrolled_done=rng.random(T) < 0.3,
                    unrolled_behavior_policy=rng.random((T, A)).astype(np.float32),
                    unrolled_action=rng.integers(0, A, T).astype(np.int32),
                    unrolled_previous_action=rng.integers(0, A, T).astype(np.int32),
                    unrolled_previous_h=rng.standard_normal((T, L)).astype(np.float32),
                    unrolled_previous_c=rng.standard_normal((T, L)).astype(np.float32))

    recs = [rec() for _ in range(7)]

    def compute():
        ref = ref_exec.load(("distributed_queue.buffer_queue",), float_dtype=torch.float64)
        rq = ref["distributed_queue.buffer_queue"].FIFOQueue(T, shape, A, cap, batch, 2, L)
        rq.set_session(ref.tf.Session())
        for i, r in enumerate(recs):
            rq.append_to_queue(task=i % 2, **r)
        d = {"size_full": np.array(rq.get_size())}
        for j in range(2):
            rb = rq.sample_batch()
            d["fields%d" % j] = np.array(rb._fields)
            d.update({"b%d/%s" % (j, n): np.stack(getattr(rb, n)) for n in FIFO_FIELDS})
        d["size_after"] = np.array(rq.get_size())
        return d

    d = reference("fifo_queue", compute)
    try:
        from distributed_reinforcement_learning_b200.distributed_queue import buffer_queue
        ours = buffer_queue.FIFOQueue(T, shape, A, cap, batch, 2, L, pinned=False)
    except Exception:                                   # library not built: the reference-side half still runs
        ours = None
    if ours is not None:
        for i, r in enumerate(recs):
            ours.append_to_queue(task=i % 2, **r)
    assert int(d["size_full"]) == 7 and (ours is None or ours.get_size() == 7)
    for j, lo in enumerate((0, 3)):
        assert tuple(str(x) for x in d["fields%d" % j]) == FIFO_FIELDS
        rb = sub(d, "b%d" % j)
        for i in range(batch):
            np.testing.assert_array_equal(rb["state"][i], recs[lo + i]["unrolled_state"])
            np.testing.assert_array_equal(rb["previous_c"][i], recs[lo + i]["unrolled_previous_c"])
        if ours is not None:
            ob = ours.sample_batch()
            for name in ("state", "reward", "done", "behavior_policy", "action", "previous_action", "previous_h",
                         "previous_c"):
                np.testing.assert_array_equal(np.stack(getattr(ob, name)), rb[name], err_msg=name)
    assert int(d["size_after"]) == 1


def test_learner_loop_call_pattern_on_the_executed_reference():
    """train_impala.py:93-113 replayed with the reference's own FIFOQueue and Agent (over the shim): gate on
    size > 3*batch, sample_batch, np.stack of every field, Agent.train; scalars equal the oracle fed the same stacks."""
    B, T, A, L = 2, 5, 6, 256
    params = it.init_params(0, torch.float32, num_action=A)
    big = synthetic.make_batch(3 * B + 1 + B, T=T, A=A, seed=77)

    def stacks(batch):
        return dict(state=np.stack(batch.state), reward=np.stack(batch.reward), action=np.stack(batch.action),
                    done=np.stack(batch.done), behavior_policy=np.stack(batch.behavior_policy),
                    previous_action=np.stack(batch.previous_action), initial_h=np.stack(batch.previous_h),
                    initial_c=np.stack(batch.previous_c))

    def compute():
        R = ref_exec.ReferenceImpala(params, trajectory=T, num_action=A)          # fresh graph with the learner agent
        queue = R.ref["distributed_queue.buffer_queue"].FIFOQueue(T, [84, 84, 4], A, 128, B, 1, L)
        queue.set_session(R.sess)
        for i in range(big["state"].shape[0]):
            queue.append_to_queue(task=0, unrolled_state=big["state"][i], unrolled_next_state=big["state"][i],
                                  unrolled_reward=big["reward"][i], unrolled_done=big["done"][i],
                                  unrolled_behavior_policy=big["behavior_policy"][i], unrolled_action=big["action"][i],
                                  unrolled_previous_action=big["previous_action"][i],
                                  unrolled_previous_h=big["initial_h"][i], unrolled_previous_c=big["initial_c"][i])
        d, steps = {}, 0
        while queue.get_size() > 3 * B:
            kw = stacks(queue.sample_batch())
            # which records the batch holds (the frames identify them), so that the oracle can be fed the same stacks
            d["rows%d" % steps] = np.array([next(i for i in range(big["state"].shape[0])
                                                 if np.array_equal(big["state"][i], s)) for s in kw["state"]])
            for k, v in kw.items():
                assert np.array_equal(v, big[k][d["rows%d" % steps]]), k
            d["got%d" % steps] = np.array(R.agent.train(**kw)[:3], np.float64)
            steps += 1
        d["steps"], d["size_after"] = np.array(steps), np.array(queue.get_size())
        return d

    d = reference("learner_loop", compute)
    O = it.Learner(params, torch.float64, "dedup", trajectory=T, num_action=A)
    assert int(d["steps"]) == 2 and int(d["size_after"]) == 3 * B - 1
    for step in range(2):
        rows = d["rows%d" % step]
        assert list(rows) == list(range(step * B, step * B + B))          # FIFO order
        exp = O.train(**{k: big[k][rows] for k in synthetic.TRAIN_FIELDS})
        for a, b in zip(d["got%d" % step], exp[:3]):
            assert abs(a - b) <= 1e-9 * max(abs(b), 1.0)


# ---- next rows: Ape-X and R2D2 agents executed -------------------------------------------------------------------
APEX_FETCH = ("main_q_value", "next_main_q_value", "target_q_value", "target_value", "state_action_value", "value_loss",
              "next_action")


def test_apex_executed_reference_equals_restatement():
    from oracle import apex_torch as ax
    A = 4
    b = ax.make_transitions(3, A=A, seed=1357)
    p, tp = ax.init_params(0, torch.float32, num_action=A), ax.init_params(1, torch.float32, num_action=A)
    args = [b[k] for k in ax.TRAIN_FIELDS]

    def compute():
        R = ref_exec.ReferenceApex(p, tp, num_action=A)
        f = R.fetch(args, list(APEX_FETCH))
        d = {"f/" + k: f[k] for k in APEX_FETCH}
        d.update({"g/" + n: v for n, v in R.gradients(R.feed(*args)).items()})
        d["td_single"] = np.asarray(R.agent.get_td_error(*args[:6]))
        for i in range(3):
            r = R.agent.distributed_train(*args)
            d["loss%d" % i], d["td%d" % i] = np.array(r[0]), np.asarray(r[1])
        d.update({"p/" + n: v for n, v in R.params().items()})
        m, v = R.adam_slots()
        d.update({"m/" + n: x for n, x in m.items()})
        d.update({"v/" + n: x for n, x in v.items()})
        d["target_differs"] = np.array(any(np.any(R.target_params()[n] != R.params()[n]) for n in R.var))
        R.agent.target_to_main()                          # despite the name: target <- main (utils.py:27-32)
        d["target_equals_main_after"] = np.array(all(np.array_equal(R.target_params()[n], R.params()[n]) for n in R.var))
        d.update({"t/" + n: v for n, v in R.target_params().items()})
        return d

    d = reference("apex", compute)
    f, rg = sub(d, "f"), sub(d, "g")
    L = ax.Learner(p, tp, torch.float64, num_action=A)
    out, g = L.gradients(*args[:6], is_weight=args[6])
    for k, ok in (("main_q_value", "main_q"), ("next_main_q_value", "next_main_q"), ("target_q_value", "target_q"),
                  ("target_value", "target_value"), ("state_action_value", "state_action_value"),
                  ("value_loss", "value_loss")):
        assert _rel(out[ok].detach().numpy(), f[k]) < 1e-12, k
    assert np.array_equal(f["next_action"], out["next_action"].numpy())
    assert len(rg) == 22                                  # target variables receive no gradient (None in TF)
    for n in g:
        assert _rel(g[n].numpy(), rg[n]) < 1e-11, n
    assert _rel(L.get_td_error(*args[:6]), d["td_single"]) < 1e-12
    for i in range(3):
        r2 = L.distributed_train(*args)
        assert float(d["loss%d" % i]) == pytest.approx(r2[0], rel=1e-6) and _rel(d["td%d" % i], r2[1]) < 1e-6
    for n, v in sub(d, "p").items():
        assert _rel(L.params[n].detach().numpy(), v) < 1e-6, n
    m, v = sub(d, "m"), sub(d, "v")
    assert max(_rel(L.m[n].numpy(), m[n]) for n in m) < 1e-5 and max(_rel(L.v[n].numpy(), v[n]) for n in v) < 1e-5
    assert bool(d["target_differs"]) and bool(d["target_equals_main_after"])
    L.target_to_main()
    for n, v in sub(d, "t").items():
        assert _rel(L.target[n].numpy(), v) < 1e-6, n


R2D2_FETCH = ("main_q", "target_q", "target_value", "state_action_value", "value_loss")


def test_r2d2_executed_reference_equals_restatement():
    from oracle import r2d2_torch as rt
    S, bi = 6, 2
    b = rt.make_sequences(2, S=S, seed=2468)
    p, tp = rt.init_params(0, torch.float32), rt.init_params(1, torch.float32)
    args = [b[k] for k in rt.TRAIN_FIELDS]

    def compute():
        R = ref_exec.ReferenceR2D2(p, tp, seq_len=S, burn_in=bi)
        f = R.fetch(args, list(R2D2_FETCH))
        d = {"f/" + k: f[k] for k in R2D2_FETCH}
        d.update({"g/" + n: v for n, v in R.gradients(R.feed(*args)).items()})
        for i in range(3):
            r = R.agent.train(*args)
            d["loss%d" % i], d["td%d" % i] = np.array(r[0]), np.asarray(r[1])
        d.update({"p/" + n: v for n, v in R.params().items()})
        R.agent.main_to_target()
        d["target_equals_main_after"] = np.array(all(np.array_equal(R.target_params()[n], R.params()[n]) for n in R.var))
        return d

    d = reference("r2d2", compute)
    f, rg = sub(d, "f"), sub(d, "g")
    L = rt.Learner(p, tp, torch.float64, seq_len=S, burn_in=bi)
    out, g = L.gradients(*args[:7], weight=args[7])
    for k in R2D2_FETCH:
        assert _rel(out[k].detach().numpy(), f[k]) < 1e-12, k
    assert len(rg) == 18
    for n in g:
        assert _rel(g[n].numpy(), rg[n]) < 1e-11, n
    for i in range(3):
        r2 = L.train(*args)
        assert float(d["loss%d" % i]) == pytest.approx(r2[0], rel=1e-6) and _rel(d["td%d" % i], r2[1]) < 1e-5
    for n, v in sub(d, "p").items():
        assert _rel(L.params[n].detach().numpy(), v) < 1e-6, n
    assert bool(d["target_equals_main_after"])
    L.main_to_target()
    for n in L.params:
        assert np.array_equal(L.target[n].numpy(), L.params[n].detach().numpy()), n


# ---- distributed_queue/buffer_queue.py:326-415 SumTree / Memory: plain NumPy in the reference -> executed as is -----
def test_reference_sumtree_and_memory_executed_equal_restatement_and_native():
    """The reference's prioritized replay memory has no TF in it: its own ``SumTree`` / ``Memory`` classes are executed
    (CPython ``random`` seeded) against ``oracle.per_np`` and -- when the library is built -- the ``drl_per_*`` mirror,
    over a wrap-around fill, interleaved priority updates and 40 ``sample`` calls: tree nodes, sampled tree indices,
    data and the beta schedule bit for bit, importance weights bit for bit (NumPy) / to 1 ulp (libm ``pow`` in csrc/per.cu)."""
    import random

    from oracle import per_np
    cap, n = 37, 8
    rng = np.random.default_rng(11)
    fill = [float(abs(rng.standard_normal()) * 3) for _ in range(cap + 9)]   # wraps: the 9 oldest records are overwritten
    upd_rng = np.random.default_rng(12)

    def compute():
        ref = ref_exec.load(("distributed_queue.buffer_queue",), float_dtype=torch.float64)
        rmem = ref["distributed_queue.buffer_queue"].Memory(cap)
        for i, e in enumerate(fill):
            rmem.add(e, ("rec", i))
        d = {"tree0": np.array(rmem.tree.tree), "n_entries": np.array(rmem.tree.n_entries),
             "write": np.array(rmem.tree.write)}
        urng = np.random.default_rng(12)
        for it_ in range(40):
            random.seed(1000 + it_)
            rbatch, ridx, rw = rmem.sample(n)
            d["idx%d" % it_], d["w%d" % it_], d["beta%d" % it_] = np.array(ridx), np.asarray(rw), np.array(rmem.beta)
            d["rec%d" % it_] = np.array([r[1] for r in rbatch])
            for j in ridx[::2]:                         # the learner writes new |td| back (train_apex.py:121-124)
                rmem.update(j, float(abs(urng.standard_normal())))
            d["tree%d" % (it_ + 1)], d["total%d" % it_] = np.array(rmem.tree.tree), np.array(rmem.tree.total())
        return d

    d = reference("sumtree_memory", compute)
    omem = per_np.MemoryNP(cap)
    try:
        from distributed_reinforcement_learning_b200.distributed_queue import buffer_queue
        nmem = buffer_queue.Memory(cap)
    except Exception:
        nmem = None
    for i, e in enumerate(fill):
        omem.add(e)
        if nmem is not None:
            nmem.add(e, ("rec", i))
    np.testing.assert_array_equal(d["tree0"], omem.tree.nodes)
    assert int(d["n_entries"]) == omem.tree.n_entries == cap and int(d["write"]) == 9
    for it_ in range(40):
        ridx, rw = [int(x) for x in d["idx%d" % it_]], d["w%d" % it_]
        rbatch = [("rec", int(x)) for x in d["rec%d" % it_]]
        random.seed(1000 + it_)
        u = [random.random() for _ in range(n)]
        oidx, odata, oprio, ow = omem.sample(n, u)
        assert list(oidx) == ridx and float(d["beta%d" % it_]) == omem.beta == pytest.approx(
            min(1.0, 0.4 + 0.001 * (it_ + 1)), abs=1e-15)
        np.testing.assert_array_equal(ow, rw)
        assert [("rec", int(j) + (cap if int(j) < 9 else 0)) for j in odata] == rbatch
        if nmem is not None:
            nbatch, nidx, nw = nmem.sample(n, u)
            assert nidx == ridx and nbatch == rbatch and nmem.beta == omem.beta
            np.testing.assert_allclose(nw, rw, rtol=4e-16, atol=0)   # libm pow vs NumPy's SIMD pow: <= 1 ulp
        for j in ridx[::2]:
            e = float(abs(upd_rng.standard_normal()))
            omem.update(j, e)
            if nmem is not None:
                nmem.update(j, e)
        np.testing.assert_allclose(d["tree%d" % (it_ + 1)], omem.tree.nodes, rtol=0, atol=0)
        assert float(d["total%d" % it_]) == omem.tree.total()
        if nmem is not None:
            assert nmem.tree.total() == omem.tree.total()


# ---- agent/a3c.py + model/actor_critic.py + optimizer/a2c.py (the fourth learner family) ---------------------------
A3C_FETCH = ("policy", "value", "next_value", "pi_loss", "baseline_loss", "entropy", "total_loss")


@pytest.mark.parametrize("clipping", ["abs_one", "soft_asymmetric"])
def test_a3c_executed_reference_equals_restatement(clipping):
    from oracle import a3c_torch as a3
    A = 5
    b = a3.make_transitions(4, A=A, seed=97)
    b["reward"] = (b["reward"] * 3).astype(np.float32)            # both branches of either clipping
    p = a3.init_params(0, torch.float32, num_action=A)
    args = [b[k] for k in a3.TRAIN_FIELDS]

    def compute():
        R = ref_exec.ReferenceA3C(p, num_action=A, reward_clipping=clipping)
        f = R.fetch(args, list(A3C_FETCH))
        d = {"f/" + k: np.asarray(f[k]) for k in A3C_FETCH}
        d.update({"g/" + n: v for n, v in R.gradients(args).items()})
        for i in range(3):
            d["train%d" % i] = np.array([float(x) for x in R.agent.train(*args)], np.float64)
        d.update({"p/" + n: v for n, v in R.params().items()})
        m, v = R.adam_slots()
        d.update({"m/" + n: x for n, x in m.items()})
        d.update({"v/" + n: x for n, x in v.items()})
        return d

    d = reference("a3c_%s" % clipping, compute)
    f, rg = sub(d, "f"), sub(d, "g")
    L = a3.Learner(p, torch.float64, num_action=A, reward_clipping=clipping)
    out = L.losses(*args)
    for k in ("policy", "value", "next_value"):
        assert _rel(out[k].detach().numpy(), f[k]) < 1e-12, k
    for k in ("pi_loss", "baseline_loss", "entropy", "total_loss"):
        assert float(out[k].detach()) == pytest.approx(float(f[k]), rel=1e-12), k
    names = list(L.params)
    g = torch.autograd.grad(out["total_loss"], [L.params[n] for n in names], allow_unused=True)
    assert len(rg) == 22
    for n, gi in zip(names, g):
        assert _rel(gi.numpy(), rg[n]) < 1e-11, n
    # three Agent.train calls: poly-decay lr, clip_by_global_norm 40, Adam with float32 beta powers
    for i in range(3):
        r2 = L.train(*args)
        for x, y in zip(d["train%d" % i], r2):
            assert float(x) == pytest.approx(float(y), rel=1e-6, abs=1e-12)
    for n, v in sub(d, "p").items():
        assert _rel(L.params[n].detach().numpy(), v) < 1e-6, n
    m, v = sub(d, "m"), sub(d, "v")
    assert max(_rel(L.m[n].numpy(), m[n]) for n in m) < 1e-5 and max(_rel(L.v[n].numpy(), v[n]) for n in v) < 1e-5
