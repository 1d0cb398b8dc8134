"""CPU self-check of the per-kernel references (tests/layer_parity.py): fed the float64 oracle's own intermediates in
device row order, every reference reproduces the oracle's activations, its activation gradients and all 24 parameter
gradients to 1e-10.  A failure of tests/test_gpu_layer_local.py therefore cannot come from a wrong reference."""
import numpy as np
import pytest
import torch

import layer_parity as lp
import parity
from oracle import impala_torch as it
from oracle import synthetic

TOL = 1e-10
# buffers the oracle does not tap: taken from the references themselves, in dependency order (a fixed point after as
# many passes as the chain is deep)
DERIVED = ("e1", "emb", "gates", "hid1", "hid2", "dlogits", "dv", "dhid2", "dhid1", "dh_part", "dz", "du")


def _params(A, seed=7):
    """glorot kernels with small non-zero biases (every bias path is exercised)."""
    p = it.init_params(0, torch.float64, num_action=A)
    g = torch.Generator().manual_seed(seed)
    for k in p:
        if k.endswith(".b"):
            p[k] = (torch.rand(p[k].shape, generator=g, dtype=torch.float64) - 0.5) * 0.1
    return p


def _oracle_buffers(out, B, T, A):
    """The oracle's taps / activation gradients in device layout (time-major rows, backward rows first Mb)."""
    tp, ag = out["taps"], out["act_grads"]
    M, Mb = B * T, B * (T - 2)

    def tm(x, shp):
        return lp.time_major(x.detach().numpy().reshape((B, T) + shp))
    buf = {"a1": tm(tp["a1"], (20, 20, 32)), "a2": tm(tp["a2"], (9, 9, 64)), "a3": tm(tp["a3"], (7, 7, 64)).reshape(M, -1),
           "h1": tm(tp["h1"], (256,)), "c1": tm(tp["c1"], (256,)), "logits": tm(tp["logits"], (A,)),
           "policy": tm(tp["policy"], (A,)), "value": tm(tp["value"], ())}
    for nm, shp in (("a1", (20, 20, 32)), ("a2", (9, 9, 64)), ("a3", (7, 7, 64))):
        d = tm(ag[nm], shp)[:Mb] * (buf[nm].reshape((M,) + shp)[:Mb] > 0)
        buf["d" + nm] = d.reshape(Mb, -1) if nm == "a3" else d
    return buf


@pytest.mark.parametrize("B,T,clip", [(2, 5, "abs_one"), (3, 7, "abs_one"), (2, 5, "soft_asymmetric")])
def test_references_reproduce_oracle(B, T, clip):
    A = 6
    batch = synthetic.make_batch(B, T=T, A=A, seed=99 + B)
    params = _params(A)
    cfg = dict(trajectory=T, num_action=A, reward_clipping=clip)
    L = it.Learner(params, torch.float64, "dedup", **cfg)
    args = [batch[k] for k in synthetic.TRAIN_FIELDS]
    out, grads = L.gradients(*args)
    buf = _oracle_buffers(out, B, T, A)
    M, Mb = B * T, B * (T - 2)
    for k in DERIVED:
        shape = {"e1": (A, 256), "emb": (A, 256), "gates": (M, 1024), "hid1": (2, M, 256), "hid2": (2, M, 256),
                 "dlogits": (Mb, 32), "dv": (Mb, 32), "dhid2": (2, Mb, 256), "dhid1": (2, Mb, 256),
                 "dh_part": (2, Mb, 256), "dz": (Mb, 1024), "du": (Mb, 256)}[k]
        buf[k] = np.zeros(shape)
    for _ in range(len(DERIVED) + 1):
        ref = lp.references(buf, params, batch, cfg, B, T, A)
        for k in DERIVED:
            if k in ("dlogits", "dv"):
                buf[k][:, :ref[k].shape[1] if ref[k].ndim == 2 else 1] = ref[k].reshape(Mb, -1)
            else:
                buf[k] = ref[k]
    ref = lp.references(buf, params, batch, cfg, B, T, A)
    errs = {}
    # forward: each layer's reference from the oracle's input to it reproduces the oracle's output
    for k in ("a1", "a2", "a3", "h1", "c1", "logits", "policy", "value"):
        errs[k] = parity.rel_err(ref[k], buf[k])
    pa = lp.device_inputs(batch)["pa"]
    errs["emb"] = parity.rel_err(ref["emb"][pa], lp.time_major(out["taps"]["emb"].detach().numpy().reshape(B, T, 256)))
    # the gate values are the nonlinearities of the oracle's own pre-activation
    z = ref["z"]
    want = np.concatenate([1 / (1 + np.exp(-z[:, :256])), np.tanh(z[:, 256:512]), 1 / (1 + np.exp(-z[:, 512:768] - 1)),
                           1 / (1 + np.exp(-z[:, 768:]))], axis=1)
    errs["gates"] = parity.rel_err(ref["gates"], want)
    # backward: the data-gradient chain from dlogits / dv down to da1 reproduces the oracle's activation gradients
    for k in ("da3", "da2", "da1"):
        errs[k] = parity.rel_err(ref[k], buf[k])
    for n, g in grads.items():
        errs["grad/" + n] = parity.rel_err(ref[n], g.detach().numpy())
    assert len([k for k in errs if k.startswith("grad/")]) == 24
    assert all(np.abs(buf[k]).max() > 0 for k in DERIVED if k not in ("dlogits", "dv")), "a derived buffer is all zero"
    bad = {k: v for k, v in errs.items() if not v < TOL}
    assert not bad, bad


def test_block_metric_sees_a_small_wrong_tile():
    """A partial last tile whose values are 1e-3 of the tensor's maximum and off by 1e-3 of themselves: ~1e-6 of the
    tensor maximum, under every per-tensor bar, but 1e-4 of the block's floor -- the block metric reports it."""
    rng = np.random.default_rng(0)
    ref = rng.standard_normal((300, 64))
    ref[256:] *= 1e-3
    got = ref.copy()
    got[256:] *= 1.0 + 1e-3
    tens, blk, label = lp.errors("hid", got, ref)
    assert tens < 2e-6 and blk > 1e-5 and label == "r256", (tens, blk, label)
    # the floor: a block of exact zeros next to a wrong tiny value is judged against 1e-2 of the tensor maximum
    got = ref.copy()
    ref[:128] = 0.0
    got[:128] = 0.0
    got[5, 3] = 1e-9
    tens, blk, _ = lp.errors("hid", got, ref)
    assert blk == pytest.approx(1e-9 / (1e-2 * np.abs(ref).max()))
