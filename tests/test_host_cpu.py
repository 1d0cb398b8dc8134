"""CPU (no GPU needed): the C-ABI library loads and exports every symbol include/drl_b200.h declares, compute
entry points fail LOUDLY without a device (no CPU fallback), the trajectory ring (FIFOQueue replacement) keeps
FIFO order / blocks / wraps, the host-side parameter inventory agrees with the oracle's, and the product
package never imports the oracle."""
import ctypes as C
import os
import re
import threading

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol(native):
    with open(os.path.join(ROOT, "include", "drl_b200.h")) as f:
        declared = sorted(set(re.findall(r"\b(drl_[a-z0-9_]+)\s*\(", f.read())))
    assert len(declared) >= 35
    missing = [n for n in declared if not hasattr(native.lib, n)]
    assert not missing, missing
    assert set(native.EXPORTS) == set(declared), set(native.EXPORTS) ^ set(declared)
    assert b"sm_90a" in native.lib.drl_version()


def test_built_for_sm_90a_only(native):
    import subprocess
    out = subprocess.run(["cuobjdump", "-lelf", native.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs


def test_compute_fails_loudly_without_a_device(native):
    if native.device_count() > 0:
        pytest.skip("a CUDA device is present")
    from distributed_reinforcement_learning_b200.learner import NativeLearner
    with pytest.raises(native.DrlError) as ei:
        NativeLearner(batch=2, trajectory=5)
    assert "no CPU fallback" in str(ei.value)
    from distributed_reinforcement_learning_b200.optimizer import vtrace
    z = np.zeros((3, 2), np.float32)
    with pytest.raises(native.DrlError):
        vtrace.from_importance_weights(z, z, z, z, np.zeros(2, np.float32))


def test_learner_rejects_math_mode_4(native):
    """math_mode 4 is not a mode: create fails as invalid, before it looks for a device, and names the accepted modes."""
    from distributed_reinforcement_learning_b200.learner import NativeLearner
    with pytest.raises(native.DrlError) as ei:
        NativeLearner(batch=2, trajectory=5, math_mode=4)
    assert ei.value.code == native.DRL_ERR_INVALID
    msg = str(ei.value)
    for accepted in ("0 (default)", "1 (FP32 FFMA)", "2 (wgmma 3xTF32)", "3 (", "5 (wgmma with 16-bit split operands)"):
        assert accepted in msg, msg
    assert "4 (" not in msg, msg


def test_product_package_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "distributed_reinforcement_learning_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                with open(os.path.join(dp, f)) as fh:
                    src = fh.read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), os.path.join(dp, f)


def test_param_inventory_matches_oracle(native):
    from distributed_reinforcement_learning_b200.model import impala_actor_critic as m
    from oracle import impala_torch as it
    assert m.param_specs() == it.param_specs()
    assert m.param_specs(num_action=6) == it.param_specs(num_action=6)
    assert m.param_count() == 4153267
    flat = m.init_params(seed=3)
    assert flat.dtype == np.float32 and flat.size == 4153267
    parts = m.split_flat(flat)
    assert parts["lstm.w"].shape == (3648, 1024) and float(np.abs(parts["conv2.b"]).max()) == 0.0
    lim = np.sqrt(6.0 / (8 * 8 * 4 + 8 * 8 * 32))
    assert np.abs(parts["conv1.w"]).max() <= lim and np.abs(parts["conv1.w"]).max() > 0.9 * lim


def test_check_properties(native):
    from distributed_reinforcement_learning_b200 import utils
    good = dict(num_actors=2, available_action=[18, 6], env=["a", "b"], model_output=18, reward_clipping="abs_one")
    utils.check_properties(good)
    for k, v in (("model_output", 5), ("env", ["a"]), ("reward_clipping", "x"), ("num_actors", 3)):
        bad = dict(good)
        bad[k] = v
        with pytest.raises(AssertionError):
            utils.check_properties(bad)


# ---- trajectory ring ------------------------------------------------------------------------------
def _traj(i, T=5, A=4, L=8, shape=(6, 6, 2)):
    rng = np.random.default_rng(i)
    return dict(s=np.full((T, *shape), i % 256, np.uint8), ns=None, r=np.full(T, float(i), np.float32),
                d=rng.random(T) < 0.5, mu=rng.random((T, A)).astype(np.float32),
                a=np.full(T, i, np.int32), pa=np.full(T, i + 1, np.int32),
                h=rng.standard_normal((T, L)).astype(np.float32), c=rng.standard_normal((T, L)).astype(np.float32))


def _push(q, t, **kw):
    q.append_to_queue(0, t["s"], t["ns"], t["r"], t["d"], t["mu"], t["a"], t["pa"], t["h"], t["c"], **kw)


def _queue(native, cap=8, batch=4):
    from distributed_reinforcement_learning_b200.distributed_queue import buffer_queue
    return buffer_queue.FIFOQueue(5, [6, 6, 2], 4, cap, batch, 2, 8, pinned=False)


def test_ring_fifo_order_and_fields(native):
    q = _queue(native)
    q.set_session(object())
    trajs = [_traj(i) for i in range(8)]
    for t in trajs:
        _push(q, t)
    assert q.get_size() == 8
    for base in (0, 4):
        b = q.sample_batch()
        assert b._fields == ('state', 'next_state', 'reward', 'done', 'behavior_policy', 'action',
                             'previous_action', 'previous_h', 'previous_c')
        assert b.next_state is None and b.state.shape == (4, 5, 6, 6, 2) and b.done.dtype == np.bool_
        for j in range(4):
            t = trajs[base + j]
            assert np.array_equal(b.state[j], t["s"]) and np.array_equal(b.reward[j], t["r"])
            assert np.array_equal(b.done[j], t["d"]) and np.array_equal(b.behavior_policy[j], t["mu"])
            assert np.array_equal(b.action[j], t["a"]) and np.array_equal(b.previous_action[j], t["pa"])
            assert np.array_equal(b.previous_h[j], t["h"]) and np.array_equal(b.previous_c[j], t["c"])
        # the reference launcher np.stack()s each field (train_impala.py:100-108): must keep working
        assert np.stack(b.state).shape == (4, 5, 6, 6, 2)
    assert q.get_size() == 0
    q.close()


def test_ring_blocks_when_full_and_when_empty(native):
    q = _queue(native, cap=4, batch=4)          # 2 batch slots
    with pytest.raises(native.TimeoutError_):
        q.sample_batch(timeout_ms=20)            # empty: fewer than batch trajectories
    for i in range(8):
        _push(q, _traj(i))
    with pytest.raises(native.TimeoutError_):
        _push(q, _traj(99), timeout_ms=20)       # both slots full
    b = q.sample_batch()
    assert int(b.action[0, 0]) == 0
    with pytest.raises(native.TimeoutError_):
        _push(q, _traj(99), timeout_ms=20)       # slot 0 is held by the consumer, slot 1 is full
    b = q.sample_batch()                         # releases slot 0
    assert int(b.action[0, 0]) == 4
    _push(q, _traj(8), timeout_ms=200)
    assert q.get_size() == 1
    q.close()


def test_ring_concurrent_producers_wrap_around(native):
    q = _queue(native, cap=8, batch=4)
    n_prod, per = 4, 12

    def prod(k):
        for i in range(per):
            _push(q, _traj(k * 100 + i))
    th = [threading.Thread(target=prod, args=(k,)) for k in range(n_prod)]
    for t in th:
        t.start()
    seen = []
    for _ in range(n_prod * per // 4):
        b = q.sample_batch(timeout_ms=5000)
        for j in range(4):
            i = int(b.action[j, 0])
            assert int(b.previous_action[j, 0]) == i + 1 and int(b.state[j, 0, 0, 0, 0]) == i % 256
            seen.append(i)
    for t in th:
        t.join()
    assert sorted(seen) == sorted(k * 100 + i for k in range(n_prod) for i in range(per))
    for k in range(n_prod):                      # per-producer order is preserved (FIFO)
        mine = [i for i in seen if i // 100 == k]
        assert mine == sorted(mine)
    q.close()


def test_ring_rejects_bad_shapes(native):
    q = _queue(native)
    t = _traj(0)
    t["r"] = np.zeros(4, np.float32)
    with pytest.raises(ValueError):
        _push(q, t)
    from distributed_reinforcement_learning_b200.distributed_queue import buffer_queue
    with pytest.raises(native.DrlError):
        buffer_queue.FIFOQueue(5, [6, 6, 2], 4, 8, 0, 2, 8, pinned=False)
    q.close()


def test_agent_constructor_surface(native):
    """Same 14 kwargs as impala.Agent (agent/impala.py:11-14, train_impala.py:48-62); no device work yet."""
    import inspect
    from distributed_reinforcement_learning_b200.agent import impala
    names = list(inspect.signature(impala.Agent.__init__).parameters)[1:]
    assert names == ["trajectory", "input_shape", "num_action", "lstm_hidden_size", "discount_factor",
                     "start_learning_rate", "end_learning_rate", "learning_frame", "baseline_loss_coef",
                     "entropy_coef", "gradient_clip_norm", "reward_clipping", "model_name", "learner_name"]
    a = impala.Agent(20, [84, 84, 4], 18, 256, 0.99, 6e-4, 0.0, 1e9, 1.0, 0.05, 40.0, "abs_one", "learner", "learner")
    for m in ("set_session", "train", "get_policy_and_action", "parameter_sync", "save_weights", "load_weights"):
        assert callable(getattr(a, m))
    with pytest.raises(AssertionError):
        impala.Agent(20, [84, 84, 4], 18, 256, 0.99, 6e-4, 0.0, 1e9, 1.0, 0.05, 40.0, "bogus", "x", "learner")
    a.set_session(None)
    assert a._params.size == 4153267 and float(a._ms.min()) == 1.0


def test_agent_checkpoint_roundtrip(native, tmp_path):
    from distributed_reinforcement_learning_b200.agent import impala
    kw = dict(trajectory=20, input_shape=[84, 84, 4], num_action=18, lstm_hidden_size=256, discount_factor=0.99,
              start_learning_rate=6e-4, end_learning_rate=0.0, learning_frame=1e9, baseline_loss_coef=1.0,
              entropy_coef=0.05, gradient_clip_norm=40.0, reward_clipping="abs_one", learner_name="learner")
    a = impala.Agent(model_name="learner", **kw)
    a.set_session(None)
    a._step = 7
    a.save_weights(str(tmp_path / "ckpt"))
    b = impala.Agent(model_name="actor_0", **kw)
    b.set_session(None)
    assert not np.array_equal(a._params, b._params)
    b.load_weights(str(tmp_path / "ckpt"))
    assert np.array_equal(a._params, b._params) and b._step == 7
    c = impala.Agent(model_name="actor_1", **kw)
    c.set_session(None)
    c.parameter_sync()                               # learner -> actor copy (utils.py:6-22)
    assert np.array_equal(c._params, a._params)


def test_shard_range(native):
    from distributed_reinforcement_learning_b200.learner import shard_range
    assert [shard_range(r, 8, 256) for r in (0, 7)] == [(0, 32), (224, 256)]
    with pytest.raises(ValueError):
        shard_range(0, 3, 32)


def test_summary_writer_writes_tensorboard_event_files(tmp_path):
    """tensorboardX.SummaryWriter stand-in (train_impala.py:91,109-113): TFRecord framing with masked CRC-32C and a
    hand-encoded Event/Summary protobuf; cross-checked against google.protobuf's wire decoder when available."""
    from distributed_reinforcement_learning_b200 import summary
    assert summary.crc32c(b"123456789") == 0xE3069283                      # CRC-32C check value
    w = summary.SummaryWriter(str(tmp_path / "runs" / "learner"))
    vals = [("data/pi_loss", -1.25, 1), ("data/baseline_loss", 3.5, 1), ("data/learning_rate", 6e-4, 2 ** 33 + 5)]
    for tag, v, st in vals:
        w.add_scalar(tag, v, st)
    w.close()
    got = summary.read_scalars(w.path)
    assert [(t, s) for t, _, s, _ in got] == [(t, s) for t, _, s in vals]
    assert [v for _, v, _, _ in got] == pytest.approx([np.float32(v) for _, v, _ in vals])
    raw = open(w.path, "rb").read()
    bad = bytearray(raw)
    bad[-6] ^= 1                                                            # flip one payload bit -> CRC must catch it
    p2 = tmp_path / "bad"
    p2.write_bytes(bytes(bad))
    with pytest.raises(ValueError):
        summary.read_scalars(str(p2))
    try:
        from google.protobuf.internal import decoder
    except Exception:
        return
    payload = summary.encode_scalar_event("data/x", 2.0, 7, 123.5)
    key, pos = decoder._DecodeVarint(payload, 0)
    assert key == (1 << 3) | 1                                              # field 1, 64-bit: wall_time


def test_unrolled_trajectory_feeds_the_ring(native):
    """utils.UnrolledTrajectory (utils.py:80-119) -> FIFOQueue.append_to_queue (train_impala.py:165-189)."""
    from distributed_reinforcement_learning_b200 import utils
    from distributed_reinforcement_learning_b200.distributed_queue import buffer_queue
    T, A, L = 4, 3, 256
    q = buffer_queue.FIFOQueue(T, [84, 84, 4], A, 4, 2, 1, L, pinned=False)
    rng = np.random.default_rng(0)
    traj = utils.UnrolledTrajectory()
    sent = []
    for ep in range(2):
        traj.initialize()
        for t in range(T):
            traj.append(state=rng.integers(0, 256, (84, 84, 4), dtype=np.uint8), next_state=None, reward=float(t),
                        done=(t == T - 1), action=t % A, behavior_policy=np.full(A, 1.0 / A, np.float32),
                        previous_action=(t + 1) % A, initial_h=np.zeros(L, np.float32), initial_c=np.ones(L, np.float32))
        u = traj.extract()
        assert list(u) == ['state', 'next_state', 'reward', 'done', 'action', 'behavior_policy', 'previous_action',
                           'initial_h', 'initial_c']
        q.append_to_queue(task=0, unrolled_state=u['state'], unrolled_next_state=u['next_state'],
                          unrolled_reward=u['reward'], unrolled_done=u['done'],
                          unrolled_behavior_policy=u['behavior_policy'], unrolled_action=u['action'],
                          unrolled_previous_action=u['previous_action'], unrolled_previous_h=u['initial_h'],
                          unrolled_previous_c=u['initial_c'])
        sent.append(u)
    assert q.get_size() == 2
    b = q.sample_batch()
    assert np.array_equal(b.state[1], np.stack(sent[1]['state'])) and b.reward[0].tolist() == [0.0, 1.0, 2.0, 3.0]
    assert b.done[:, -1].all() and b.previous_c.min() == 1.0
    q.close()


def test_record_queues_and_actor_buffers(native):
    """In-process stand-ins of ApexFIFOQueue / R2D2FIFOQueue / A3CFIFOQueue (bounded, blocking, FIFO, static shapes) and
    of the actor-side LocalBuffer / R2D2TrajectoryBuffer (distributed_queue/buffer_queue.py:7-318)."""
    from distributed_reinforcement_learning_b200.distributed_queue import buffer_queue as bq
    T, shape = 3, [84, 84, 4]
    q = bq.ApexFIFOQueue(trajectory=T, input_shape=shape, output_size=4, queue_size=2, batch_size=32, num_actors=1)
    q.set_session(object())
    rec = lambda v: dict(unrolled_state=np.full((T, *shape), v, np.uint8), unrolled_next_state=np.zeros((T, *shape), np.uint8),
                         unrolled_previous_action=np.zeros(T, np.int32), unrolled_action=np.full(T, v, np.int32),
                         unrolled_reward=np.zeros(T, np.float32), unrolled_done=np.zeros(T, bool))
    q.append_to_queue(task=0, **rec(1))
    q.append_to_queue(task=0, **rec(2))
    assert q.get_size() == 2
    with pytest.raises(native.TimeoutError_):
        q.append_to_queue(task=0, timeout=0.05, **rec(3))                 # full -> blocks (tf.FIFOQueue)
    with pytest.raises(ValueError):
        q.append_to_queue(task=0, **dict(rec(3), unrolled_reward=np.zeros(T + 1, np.float32)))   # static placeholder shapes
    got = []
    th = threading.Thread(target=lambda: got.append(q.sample_batch(3)))   # waits for the third record
    th.start()
    q.append_to_queue(task=0, timeout=2.0, **rec(3))
    th.join(5)
    b = got[0]
    assert b._fields == ('state', 'next_state', 'previous_action', 'action', 'reward', 'done')
    assert [int(a[0]) for a in b.action] == [1, 2, 3] and q.get_size() == 0   # FIFO order
    r = bq.R2D2FIFOQueue(seq_len=T, input_shape=[84, 84, 1], output_size=4, queue_size=4, batch_size=2, num_actors=1, lstm_size=64)
    for v in (5, 6):
        r.append_to_queue(0, np.zeros((T, 84, 84, 1), np.uint8), np.zeros(T, np.int32), np.full(T, v, np.int32),
                          np.zeros(T, np.float32), np.zeros(T, bool), np.zeros((T, 64), np.float32), np.zeros((T, 64), np.float32))
    rb = r.sample_batch()
    assert rb._fields[-2:] == ('previous_h', 'previous_c') and [int(a[0]) for a in rb.action] == [5, 6]
    a = bq.A3CFIFOQueue(trajectory_size=T, input_shape=shape, output_size=4, num_actors=1)
    a.append_to_queue(0, *[rec(7)[k] for k in ("unrolled_state", "unrolled_next_state", "unrolled_previous_action",
                                              "unrolled_action", "unrolled_reward", "unrolled_done")])
    ab = a.sample_batch()
    assert len(ab.state) == 1 and ab.state[0].shape == (T, 84, 84, 4) and a.get_size() == 0
    with pytest.raises(native.TimeoutError_):
        a.sample_batch(timeout=0.05)                                      # empty -> blocks
    # a time-out in the middle of a batch loses nothing: the records already taken go back to the front, in order
    for v in (8, 9):
        r.append_to_queue(0, np.zeros((T, 84, 84, 1), np.uint8), np.zeros(T, np.int32), np.full(T, v, np.int32),
                          np.zeros(T, np.float32), np.zeros(T, bool), np.zeros((T, 64), np.float32), np.zeros((T, 64), np.float32))
    r.batch_size = 3
    with pytest.raises(native.TimeoutError_):
        r.sample_batch(timeout=0.05)
    assert r.get_size() == 2
    r.batch_size = 2
    assert [int(x[0]) for x in r.sample_batch().action] == [8, 9]
    lb = bq.LocalBuffer(capacity=5)
    for i in range(8):
        lb.append(i, i + 1, 0, 1, float(i), False)
    assert len(lb) == 5 and list(lb.state) == [3, 4, 5, 6, 7]
    s = lb.sample(3)
    assert len(s["state"]) == 3 and len(set(s["state"])) == 3 and all(ns == st + 1 for st, ns in zip(s["state"], s["next_state"]))
    tb = bq.R2D2TrajectoryBuffer(seq_len=4)
    for i in range(6):
        tb.append(i, 0, 1, 0.0, False, np.zeros(64), np.ones(64))
    ex = tb.extract()
    assert list(ex["state"]) == [2, 3, 4, 5] and set(ex) == {'state', 'previous_action', 'action', 'reward', 'done', 'initial_h', 'initial_c'}
    tb.init()
    assert len(tb) == 0


def test_unrolled_a3c_trajectory(native):
    from distributed_reinforcement_learning_b200 import utils
    t = utils.UnrolledA3CTrajectory()
    t.initialize()
    for i in range(3):
        t.append(state=np.full((2, 2), i), next_state=np.full((2, 2), i + 1), previous_action=i, action=i + 1, reward=0.5 * i,
                 done=(i == 2))
    d = t.extract()
    assert set(d) == {'state', 'next_state', 'previous_action', 'action', 'reward', 'done'}
    assert d['state'].shape == (3, 2, 2) and d['action'].tolist() == [1, 2, 3] and d['done'].tolist() == [False, False, True]
    t.initialize()
    assert len(t.unroll_data.state) == 0


def test_ctypes_structs_match_the_c_header(native, tmp_path):
    """ABI drift guard: sizeof / offsetof of every struct of include/drl_b200.h as gcc lays them out must equal the
    ctypes mirror in _native.py (a mismatch would silently scramble a configuration)."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    N = native
    pairs = [("drl_learner_config", N.LearnerConfig), ("drl_step_out", N.StepOut), ("drl_ring_batch", N.RingBatch),
             ("drl_apex_config", N.ApexConfig), ("drl_apex_out", N.ApexOut), ("drl_a3c_config", N.A3cConfig),
             ("drl_a3c_out", N.A3cOut), ("drl_r2d2_config", N.R2d2Config), ("drl_r2d2_out", N.R2d2Out)]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "drl_b200.h"', 'int main(void) {']
    for cname, ct in pairs:
        lines.append('  printf("%s size %%zu\\n", sizeof(%s));' % (cname, cname))
        for fname, _ in ct._fields_:
            lines.append('  printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (cname, fname, cname, fname))
    lines += ['  return 0;', '}']
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "abi"
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
    subprocess.run(["gcc", "-std=c99", "-I", inc, str(src), "-o", str(exe)], check=True, capture_output=True)
    got = dict(ln.rsplit(" ", 1) for ln in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    for cname, ct in pairs:
        assert int(got["%s size" % cname]) == C.sizeof(ct), cname
        for fname, _ in ct._fields_:
            assert int(got["%s.%s" % (cname, fname)]) == getattr(ct, fname).offset, (cname, fname)


def test_docs_name_only_real_entry_points(native):
    """Every drl_* name that DESIGN.md / INTEGRATION.md / README.md mention is exported by the library (wildcards like
    drl_ring_* and family placeholders excluded)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exported = set(native.EXPORTS)
    prefixes = {e.rsplit("_", 1)[0] for e in exported} | {"drl_learner", "drl_apex", "drl_r2d2", "drl_a3c", "drl_per",
                                                          "drl_ring", "drl_vtrace"}
    for doc in ("DESIGN.md", "INTEGRATION.md", "README.md"):
        text = open(os.path.join(root, doc)).read()
        for name in set(re.findall(r"\bdrl_[a-z0-9_]+\b", text)):
            if name in exported or name in ("drl_b200",) or name.rstrip("_") in prefixes or name.endswith("_"):
                continue
            if name in ("drl_learner_config", "drl_step_out", "drl_apex_config", "drl_apex_out", "drl_a3c_config",
                        "drl_a3c_out", "drl_r2d2_config", "drl_r2d2_out", "drl_ring_batch", "drl_learner_peer"):
                continue
            assert any(e.startswith(name) for e in exported), "%s mentions %s, which the library does not export" % (doc, name)
