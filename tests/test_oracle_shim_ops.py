"""The TF 1.14 op semantics that ``oracle/tf1_shim`` restates (its docstring lists them) against INDEPENDENT NumPy
implementations written from TensorFlow's documented formulas -- explicit loops, no torch.  The executed-reference
tests (test_oracle_refexec.py) make every graph-construction decision the reference's own; what they cannot see is
an error in the shim's own op kernels.  This file closes that: conv2d / dense / LSTMCell / scan / one_hot / argmax /
clip_by_global_norm / polynomial_decay / RMSProp / Adam, each on small random inputs in float64."""
import importlib
import os
import sys

import numpy as np
import pytest
import torch

from oracle import ref_exec


@pytest.fixture()
def tf():
    saved_path = list(sys.path)
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k.split(".")[0] in ("tensorflow", "gym", "tensorboardX")}
    sys.path.insert(0, ref_exec.SHIM_DIR)
    try:
        mod = importlib.import_module("tensorflow")
        assert mod.__version__.endswith("-shim")
        mod._shim.FLOAT = torch.float64
        mod.reset_default_graph()
        yield mod
    finally:
        sys.path[:] = saved_path
        for k in list(sys.modules):
            if k.split(".")[0] in ("tensorflow", "gym", "tensorboardX"):
                del sys.modules[k]
        sys.modules.update(saved)


def _f32(a):
    """TF variables are float32: values that survive ``Variable.set`` unchanged."""
    return np.asarray(a, np.float32).astype(np.float64)


def _vars(tf):
    return {v.op_name: v for v in tf.trainable_variables()}


def test_conv2d_valid_nhwc_hwio_is_cross_correlation(tf):
    rng = np.random.default_rng(0)
    x = _f32(rng.standard_normal((2, 9, 8, 3)))      # float feeds are cast to float32 first, like a TF feed
    ph = tf.placeholder(tf.float32, shape=[None, 9, 8, 3])
    y = tf.layers.conv2d(inputs=ph, filters=4, kernel_size=[3, 2], strides=[2, 3], padding="VALID", activation=tf.nn.relu)
    sess = tf.Session()
    sess.run(tf.global_variables_initializer())
    v = _vars(tf)
    w = _f32(rng.standard_normal((3, 2, 3, 4)))
    b = _f32(rng.standard_normal(4))
    v["conv2d/kernel"].set(w)
    v["conv2d/bias"].set(b)
    got = sess.run(y, feed_dict={ph: x})
    OH, OW = (9 - 3) // 2 + 1, (8 - 2) // 3 + 1
    exp = np.zeros((2, OH, OW, 4))
    for n in range(2):
        for oy in range(OH):
            for ox in range(OW):
                for co in range(4):
                    acc = b[co]
                    for ky in range(3):
                        for kx in range(2):
                            for ci in range(3):
                                acc += x[n, oy * 2 + ky, ox * 3 + kx, ci] * w[ky, kx, ci, co]     # no kernel flip
                    exp[n, oy, ox, co] = max(acc, 0.0)
    assert got.shape == exp.shape
    np.testing.assert_allclose(got, exp, rtol=1e-12, atol=1e-12)
    # glorot_uniform kernel / zero bias at initialisation (tf.layers defaults)
    tf.reset_default_graph()
    ph = tf.placeholder(tf.float32, shape=[None, 9, 8, 3])
    tf.layers.conv2d(inputs=ph, filters=64, kernel_size=[3, 2], strides=[1, 1], padding="VALID")
    sess = tf.Session()
    sess.run(tf.global_variables_initializer())
    v = _vars(tf)
    k0 = v["conv2d/kernel"].numpy()
    limit = np.sqrt(6.0 / (3 * 2 * 3 + 3 * 2 * 64))
    assert np.all(np.abs(k0) <= limit) and np.abs(k0).max() > 0.9 * limit and np.all(v["conv2d/bias"].numpy() == 0)


def test_dense_flatten_one_hot_argmax(tf):
    rng = np.random.default_rng(1)
    ph = tf.placeholder(tf.float32, shape=[None, 2, 3])
    ids = tf.placeholder(tf.int32, shape=[None])
    y = tf.layers.dense(inputs=tf.layers.flatten(ph), units=5, activation=None)
    oh = tf.one_hot(ids, 4)
    am = tf.argmax(tf.layers.flatten(ph), axis=1)
    sess = tf.Session()
    sess.run(tf.global_variables_initializer())
    v = _vars(tf)
    w, b = _f32(rng.standard_normal((6, 5))), _f32(rng.standard_normal(5))
    v["dense/kernel"].set(w)
    v["dense/bias"].set(b)
    x = _f32(rng.standard_normal((3, 2, 3)))
    x[1] = 0.25                                            # all equal: argmax must return the FIRST index
    got, goh, gam = sess.run([y, oh, am], feed_dict={ph: x, ids: np.array([0, 3, 4, -1][:3] + [2][:0])})
    np.testing.assert_allclose(got, x.reshape(3, 6) @ w + b, rtol=1e-13)
    assert np.array_equal(goh, np.array([[1, 0, 0, 0], [0, 0, 0, 1], [0, 0, 0, 0]], float))   # 4 is out of range: zeros
    assert gam[1] == 0 and gam[0] == int(np.argmax(x[0].ravel()))


def test_lstm_cell_gate_order_and_forget_bias(tf):
    rng = np.random.default_rng(2)
    nin, L, Bn = 5, 3, 4
    xin = tf.placeholder(tf.float32, shape=[None, 1, nin])
    c_ph = tf.placeholder(tf.float32, shape=[None, L])
    h_ph = tf.placeholder(tf.float32, shape=[None, L])
    cell = tf.nn.rnn_cell.LSTMCell(L)
    state = tf.nn.rnn_cell.LSTMStateTuple(c_ph, h_ph)
    out, (c1, h1) = tf.nn.dynamic_rnn(cell, xin, initial_state=state, dtype=tf.float32)
    sess = tf.Session()
    sess.run(tf.global_variables_initializer())
    v = _vars(tf)
    assert set(v) == {"rnn/lstm_cell/kernel", "rnn/lstm_cell/bias"}
    W, b = _f32(rng.standard_normal((nin + L, 4 * L))), _f32(rng.standard_normal(4 * L))
    v["rnn/lstm_cell/kernel"].set(W)
    v["rnn/lstm_cell/bias"].set(b)
    x, c0, h0 = (_f32(rng.standard_normal(sh)) for sh in ((Bn, 1, nin), (Bn, L), (Bn, L)))
    g_out, g_c, g_h = sess.run([out, c1, h1], feed_dict={xin: x, c_ph: c0, h_ph: h0})
    sig = lambda z: 1.0 / (1.0 + np.exp(-z))
    z = np.concatenate([x[:, 0], h0], axis=1) @ W + b       # [inputs, h] (in that order) times the kernel
    i, j, f, o = z[:, :L], z[:, L:2 * L], z[:, 2 * L:3 * L], z[:, 3 * L:]
    c = sig(f + 1.0) * c0 + sig(i) * np.tanh(j)             # forget_bias 1.0 inside the sigmoid
    h = sig(o) * np.tanh(c)
    np.testing.assert_allclose(g_c, c, rtol=1e-12)
    np.testing.assert_allclose(g_h, h, rtol=1e-12)
    np.testing.assert_allclose(g_out[:, 0], h, rtol=1e-12)


def test_scan_reverse_and_stop_gradient(tf):
    a = tf.placeholder(tf.float32, shape=[None, 3])
    b = tf.placeholder(tf.float32, shape=[None, 3])
    init = tf.zeros_like(a[0])
    res = tf.scan(lambda acc, ab: ab[0] + ab[1] * acc, (a, b), initializer=init, reverse=True, back_prop=False)
    rng = np.random.default_rng(3)
    av, bv = _f32(rng.standard_normal((6, 3))), _f32(rng.standard_normal((6, 3)))
    got = tf.Session().run(res, feed_dict={a: av, b: bv})
    exp, acc = np.zeros((6, 3)), np.zeros(3)
    for t in range(5, -1, -1):
        acc = av[t] + bv[t] * acc
        exp[t] = acc
    np.testing.assert_allclose(got, exp, rtol=1e-13)


def test_clip_by_global_norm_and_polynomial_decay(tf):
    rng = np.random.default_rng(4)
    g1, g2 = rng.standard_normal((3, 4)) * 30, rng.standard_normal(7) * 30
    t1, t2 = tf.constant(g1), tf.constant(g2)
    clipped, norm = tf.clip_by_global_norm([t1, None, t2], 40.0)
    sess = tf.Session()
    c1, c2, n = sess.run([clipped[0], clipped[2], norm])
    gn = np.sqrt(np.sum(g1 ** 2) + np.sum(g2 ** 2))
    assert clipped[1] is None and n == pytest.approx(gn, rel=1e-13) and gn > 40
    np.testing.assert_allclose(c1, g1 * 40.0 / gn, rtol=1e-12)
    np.testing.assert_allclose(c2, g2 * 40.0 / gn, rtol=1e-12)
    small, _ = tf.clip_by_global_norm([tf.constant(g1 * 1e-3)], 40.0)
    np.testing.assert_allclose(sess.run(small[0]), g1 * 1e-3, rtol=1e-13)          # norm < clip: unchanged
    step = tf.train.get_or_create_global_step()
    lr = tf.train.polynomial_decay(6e-4, step, 1000, 1e-5)
    sess.run(tf.global_variables_initializer())
    for s in (0, 250, 1000, 5000):
        step.set(np.int64(s))
        exp = np.float32((np.float32(6e-4) - np.float32(1e-5)) * np.float32(1 - min(s, 1000) / 1000) + np.float32(1e-5))
        assert float(sess.run(lr)) == pytest.approx(float(exp), rel=1e-6)


@pytest.mark.parametrize("bad", ["nan", "inf", "overflow", "zero"])
def test_clip_by_global_norm_non_finite_and_zero_norms(tf, bad):
    """TF 1.14 clip_ops: scale = clip * min(1/norm, 1/clip) + (norm - norm).  A NaN or infinite global norm (an element
    NaN or infinite, or a sum of squares that overflows) makes every clipped tensor NaN; a zero norm leaves them as
    they are."""
    g1, g2 = np.zeros((3, 4)), np.linspace(-1.0, 1.0, 7) * (0.0 if bad == "zero" else 1.0)
    if bad == "overflow":
        g1[0, :2] = 1e155                           # each square is finite in float64, their sum is not
    elif bad != "zero":
        g1[1, 2] = float(bad)
    clipped, norm = tf.clip_by_global_norm([tf.constant(g1), None, tf.constant(g2)], 40.0)
    with np.errstate(all="ignore"):
        c1, c2, n = tf.Session().run([clipped[0], clipped[2], norm])
    if bad == "zero":
        assert n == 0.0 and np.array_equal(c1, g1) and np.array_equal(c2, g2)
    else:
        assert not np.isfinite(n) and np.isnan(c1).all() and np.isnan(c2).all()


def _quadratic(tf, w0):
    w = tf.get_variable("w", shape=list(w0.shape), initializer=tf.zeros_initializer())
    t = tf.placeholder(tf.float32, shape=list(w0.shape))
    loss = tf.reduce_sum(tf.square(w - t) * 0.5)          # gradient = w - t
    return w, t, loss


def test_rmsprop_tf1_semantics(tf):
    rng = np.random.default_rng(5)
    w0, tgt = _f32(rng.standard_normal(6)), _f32(rng.standard_normal(6))
    w, t, loss = _quadratic(tf, w0)
    opt = tf.train.RMSPropOptimizer(0.01, decay=0.99, momentum=0.0, epsilon=0.1)
    train = opt.minimize(loss)
    sess = tf.Session()
    sess.run(tf.global_variables_initializer())
    w.set(w0)
    ms, mom, wv = np.ones(6), np.zeros(6), w0.copy()       # the slot starts at ONE (RMSPropOptimizer._create_slots)
    for _ in range(3):
        g = wv - tgt
        ms = ms + (1 - 0.99) * (g * g - ms)
        mom = 0.0 * mom + 0.01 * g / np.sqrt(ms + 0.1)      # epsilon INSIDE the square root
        wv = wv - mom
        sess.run(train, feed_dict={t: tgt})
        np.testing.assert_allclose(w.numpy(), wv, rtol=1e-12)
    np.testing.assert_allclose(opt.get_slot(w, "rms").numpy(), ms, rtol=1e-12)


def test_adam_tf1_semantics(tf):
    rng = np.random.default_rng(6)
    w0, tgt = _f32(rng.standard_normal(5)), _f32(rng.standard_normal(5))
    w, t, loss = _quadratic(tf, w0)
    opt = tf.train.AdamOptimizer(1e-2)
    train = opt.minimize(loss)
    sess = tf.Session()
    sess.run(tf.global_variables_initializer())
    w.set(w0)
    m, v, wv = np.zeros(5), np.zeros(5), w0.copy()
    b1p, b2p = np.float32(0.9), np.float32(0.999)          # float32 beta-power variables, multiplied AFTER each apply
    for _ in range(4):
        g = wv - tgt
        lr_t = 1e-2 * np.sqrt(1 - float(b2p)) / (1 - float(b1p))
        m = m + (g - m) * (1 - 0.9)
        v = v + (g * g - v) * (1 - 0.999)
        wv = wv - lr_t * m / (np.sqrt(v) + 1e-8)            # epsilon OUTSIDE the square root
        b1p, b2p = np.float32(b1p * np.float32(0.9)), np.float32(b2p * np.float32(0.999))
        sess.run(train, feed_dict={t: tgt})
        np.testing.assert_allclose(w.numpy(), wv, rtol=1e-10)
    np.testing.assert_allclose(opt.get_slot(w, "m").numpy(), m, rtol=1e-12)
    np.testing.assert_allclose(opt.get_slot(w, "v").numpy(), v, rtol=1e-12)
