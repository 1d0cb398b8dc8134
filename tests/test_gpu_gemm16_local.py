"""-m gpu: the wgmma accumulators of the math-mode-5 GEMMs stay in registers.

When an accumulator is indexed at run time (an epilogue loop that is not unrolled, say) the compiler moves it to local
memory and serialises every wgmma of the main loop.  The results are the same, the LSTM data gradient alone is about a
quarter slower on an H100, and no parity test notices; this one asks the driver how much local memory three of the
step's GEMM kernels use."""
import ctypes

import pytest

pytestmark = pytest.mark.gpu

KERNELS = ("lstm_fwd", "lstm_dgrad", "lstm_wgrad")


def test_accumulators_in_registers():
    from distributed_reinforcement_learning_b200 import _native as N
    if N.device_count() < 1:
        pytest.fail("needs a CUDA device")
    out = (ctypes.c_int32 * len(KERNELS))()
    N.check(N.lib.drl_debug_gemm16_local_bytes(out))
    assert dict(zip(KERNELS, out)) == {k: 0 for k in KERNELS}
