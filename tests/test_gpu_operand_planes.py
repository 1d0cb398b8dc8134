"""-m gpu: the 16-bit operand planes of math mode 5 hold exactly the bf16 hi / lo split of their fp32 buffers.

conv2_fwd / conv3_fwd and the conv3 / conv2 data gradients copy their A tiles from planes of a1, a2, da3 and da2 that the
kernels producing those buffers write beside them.  Each plane is [hi | lo]: hi = bf16(x) and lo = bf16(x - hi), both
rounded to nearest even, in the buffer's own element order.  These are the bits the 16-bit GEMM producers would have made
from the fp32 value.  A plane that differs in one element changes the data the tensor cores see."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PLANES = {"a1": ("M", 400 * 32), "a2": ("M", 81 * 64), "da3": ("Mb", 3136), "da2": ("Mb", 81 * 64)}


def bf16_rne(x):
    """float32 array -> float32 array holding its bf16 round-to-nearest-even value (finite inputs)."""
    u = x.astype(np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(np.float32)


def split(x):
    """The [hi | lo] bf16 bit patterns of float32 x, as uint16."""
    hi = bf16_rne(x)
    lo = bf16_rne((x - hi).astype(np.float32))
    bits = lambda v: (v.view(np.uint32) >> 16).astype(np.uint16)
    return np.concatenate([bits(hi), bits(lo)])


def test_bf16_rne_matches_torch():
    import torch
    x = np.random.RandomState(0).standard_normal(4096).astype(np.float32) * np.float32(3.0)
    x[:4] = [0.0, -0.0, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8]          # ties to even, both ways
    want = torch.from_numpy(x).to(torch.bfloat16).to(torch.float32).numpy()
    assert np.array_equal(bf16_rne(x).view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("B,T", [(32, 20), (3, 5)])
def test_planes_are_the_split_of_their_buffers(B, T):
    from distributed_reinforcement_learning_b200 import _native as N
    from distributed_reinforcement_learning_b200.learner import NativeLearner
    from oracle import impala_torch as it
    from oracle import synthetic
    if N.device_count() < 1:
        pytest.fail("needs a CUDA device")
    import torch
    A = 6
    eng = NativeLearner(batch=B, trajectory=T, num_action=A, math_mode=5)
    try:
        eng.set_params(it.flatten_params(it.init_params(3, torch.float32, num_action=A)))
        b = synthetic.make_batch(B, T=T, A=A, seed=7)
        eng.stage(0, *[b[k] for k in synthetic.TRAIN_FIELDS])
        eng.step(0)
        rows = {"M": B * T, "Mb": B * (T - 2)}
        for name, (r, width) in PLANES.items():
            n = rows[r] * width
            x = eng.read_buffer(name, n)
            plane = eng.read_buffer(name + "_plane", n).view(np.uint16)
            want = split(x)
            bad = np.flatnonzero(plane != want)
            assert bad.size == 0, "%s plane: %d of %d halves differ, first at %d (got %#06x, want %#06x)" % (
                name, bad.size, want.size, bad[0], plane[bad[0]], want[bad[0]])
            assert np.count_nonzero(x) > n // 10, "%s is mostly zero: the check would be weak" % name
    finally:
        eng.close()


def test_planes_are_not_kept_outside_math_mode_5():
    from distributed_reinforcement_learning_b200 import _native as N
    from distributed_reinforcement_learning_b200.learner import NativeLearner
    if N.device_count() < 1:
        pytest.fail("needs a CUDA device")
    eng = NativeLearner(batch=2, trajectory=5, num_action=4, math_mode=2)
    try:
        with pytest.raises(N.DrlError, match="not kept"):
            eng.read_buffer("a1_plane", 2 * 5 * 400 * 32)
    finally:
        eng.close()
