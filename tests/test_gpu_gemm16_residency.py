"""-m gpu: the math-mode-5 GEMMs sized for two CTAs per SM (conv2 / conv3 forward, conv2 data gradient) get two.

Their registers are split by role (setmaxnreg) so that two CTAs of 512 threads fit in the 65,536 registers of an SM, and
their shared memory is sized for half an SM.  A change to either that pushes a kernel past half an SM computes the same
results at one CTA per SM, only slower, so no parity test would notice; this one asks the driver how many CTAs of each
kernel are resident at the block size and dynamic shared memory the library launches with."""
import ctypes

import pytest

pytestmark = pytest.mark.gpu

KERNELS = ("conv2_fwd", "conv3_fwd", "conv2_dgrad")


def test_two_ctas_per_sm():
    from distributed_reinforcement_learning_b200 import _native as N
    if N.device_count() < 1:
        pytest.fail("needs a CUDA device")
    out = (ctypes.c_int32 * len(KERNELS))()
    N.check(N.lib.drl_debug_gemm16_residency(out))
    assert dict(zip(KERNELS, out)) == {k: 2 for k in KERNELS}
