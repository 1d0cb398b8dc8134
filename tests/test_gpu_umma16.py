"""-m gpu: the wgmma f16 / bf16 contraction core with 16-bit split operands (csrc/gemm_umma16.cuh, math_mode 5).
(1) drl_debug_gemm cores 5 (bf16 split) / 6 (fp16 split) / 7, 8 (same with B from a pre-tiled K-major image fetched by
    the bulk-copy loader warp): every operand-major combination, tile width, split-K and ragged shapes against NumPy
    float64.  Expected error of hi*hi + hi*lo + lo*hi: ~2^-16 per product for bf16 (random sign: ~1e-6 .. 1e-5 of the
    largest output), ~2^-22 for fp16 (fp32-grade).
(2) the whole learner step with math_mode=5 against the float64 oracle, same 1e-4 bar as every other mode."""
import numpy as np
import pytest

import parity
from test_gpu_umma import _gemm

pytestmark = pytest.mark.gpu

TOL = {5: 2e-5, 6: 2e-6, 7: 2e-5, 8: 2e-6}


@pytest.mark.parametrize("core", [5, 6, 7, 8])
@pytest.mark.parametrize("a_km,b_km", [(1, 0), (1, 1), (0, 0), (0, 1)])
@pytest.mark.parametrize("bn", [32, 64, 128, 256])
def test_umma16_gemm_operand_majors(native, core, a_km, b_km, bn):
    if core in (5, 6) and bn == 32 and not b_km:
        pytest.skip("gathered MN-major 16-bit B tiles are built from 64-column atoms (bn >= 64)")
    err, cs = _gemm(native, core, bn, a_km, b_km, 256, 128, 192, 1)
    assert err < TOL[core], (core, a_km, b_km, bn, err)
    if cs is not None and core in (5, 6):
        assert cs < 1e-5, cs


@pytest.mark.parametrize("core", [5, 7])
@pytest.mark.parametrize("M,N,K,splits,bn", [(128, 64, 64, 1, 64), (132, 72, 104, 1, 64), (640, 1024, 3648, 4, 128),
                                             (3648, 1024, 576, 1, 256), (640, 1024, 3648, 7, 256), (52, 64, 4096, 7, 64),
                                             (1000, 200, 72, 2, 128), (300, 32, 256, 1, 32)])
@pytest.mark.parametrize("a_km,b_km", [(1, 0), (0, 0), (1, 1)])
def test_umma16_gemm_shapes_and_splitk(native, core, M, N, K, splits, bn, a_km, b_km):
    if core == 5 and bn == 32 and not b_km:
        pytest.skip("gathered MN-major 16-bit B tiles need bn >= 64")
    err, cs = _gemm(native, core, bn, a_km, b_km, M, N, K, splits, seed=M + N)
    assert err < 3e-5, (core, M, N, K, splits, bn, a_km, b_km, err)
    if cs is not None and core == 5:
        assert cs < 2e-5, cs


def _assert_all(errs):
    bad = parity.failures(errs)
    assert not bad, "parity failures (rel err): %s" % sorted(bad.items(), key=lambda kv: -kv[1])[:12]


def test_step_small_config_split16(native):
    _assert_all(parity.compare_step(4, T=20, math_mode=5))


def test_step_reference_config_split16(native):
    _assert_all(parity.compare_step(32, T=20, layers=False, math_mode=5))


@pytest.mark.parametrize("B,T,A", [(1, 3, 2), (3, 7, 6), (5, 32, 18)])
def test_step_ragged_shapes_split16(native, B, T, A):
    _assert_all(parity.compare_step(B, T=T, A=A, math_mode=5))


def test_three_steps_cuda_graph_split16(native):
    _assert_all(parity.compare_step(4, T=20, steps=3, layers=False, use_cuda_graph=True, math_mode=5))
