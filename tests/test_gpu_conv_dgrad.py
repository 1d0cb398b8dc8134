"""-m gpu: the conv3 / conv2 data gradients of the math-mode-5 IMPALA step (csrc/layers.cu, net_backward): the conv3 one
as a gather-GEMM over the input pixels, the conv2 one as a single GEMM over all four stride-2 parity classes.  Each is
checked in isolation against float64 PyTorch from the step's own inputs: da2 from the GPU's da3, da1 from the GPU's
da2, with the ReLU masks of the GPU's a2 / a1 and the parameters the step ran with.  The bar is the bf16 3-product bar
of test_gpu_umma16.py: 2e-5 of each tensor's largest magnitude."""
import numpy as np
import pytest
import torch

import parity
from oracle import impala_torch as it
from oracle import synthetic

pytestmark = pytest.mark.gpu

TOL = 2e-5


def _nchw(x_nhwc):
    return torch.from_numpy(np.ascontiguousarray(x_nhwc, dtype=np.float64)).permute(0, 3, 1, 2)


def _dgrad(dy_nhwc, w_hwio, act_nhwc, stride):
    """relu'(act) * conv_transpose(dy, w) in float64, NHWC in and out (TF VALID convolution, HWIO weights)."""
    w = w_hwio.to(torch.float64).permute(3, 2, 0, 1)   # HWIO -> OIHW
    n, h, wd, c = act_nhwc.shape
    dx = torch.nn.grad.conv2d_input((n, c, h, wd), w, _nchw(dy_nhwc), stride=stride)
    return dx.permute(0, 2, 3, 1).numpy() * (act_nhwc > 0)


@pytest.mark.parametrize("B,T,A", [(32, 20, 18), (3, 7, 6), (5, 32, 18)])
def test_conv_data_gradients_mode5(native, B, T, A):
    check_conv_data_gradients(B, T, A)


def check_conv_data_gradients(B, T, A):
    batch, params, cfg = parity.make_case(B, T, A)
    eng = parity.native_learner(batch, params, cfg, math_mode=5)
    M, Mb = B * T, B * (T - 2)
    try:
        p = it.unflatten_params(eng.get_params(), torch.float64, num_action=A)   # what the step runs with
        eng.stage(0, *[batch[k] for k in synthetic.TRAIN_FIELDS])
        eng.step(0)
        # device rows are time-major; the rows t <= T-3 that receive gradient are the first Mb of every activation
        a1 = eng.read_buffer("a1", M * 400 * 32).reshape(M, 20, 20, 32)[:Mb]
        a2 = eng.read_buffer("a2", M * 81 * 64).reshape(M, 9, 9, 64)[:Mb]
        da3 = eng.read_buffer("da3", Mb * 49 * 64).reshape(Mb, 7, 7, 64)
        da2 = eng.read_buffer("da2", Mb * 81 * 64).reshape(Mb, 9, 9, 64)
        da1 = eng.read_buffer("da1", Mb * 400 * 32).reshape(Mb, 20, 20, 32)
    finally:
        eng.close()
    assert np.abs(da3).max() > 0 and np.abs(da2).max() > 0
    for name, got, ref in (("da2", da2, _dgrad(da3, p["conv3.w"], a2, 1)),
                           ("da1", da1, _dgrad(da2, p["conv2.w"], a1, 2))):
        err = parity.rel_err(got, ref)
        assert err < TOL, (name, B, T, err)
