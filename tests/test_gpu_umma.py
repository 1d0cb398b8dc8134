"""-m gpu: the wgmma 3xTF32 contraction core (csrc/gemm_umma.cuh).
(1) drl_debug_gemm: one plain GEMM per operand-major combination (K-major / MN-major A and B -- the
    128-byte-swizzled shared-memory layouts and UMMA descriptors), tile width and split-K setting, against
    NumPy float64; the FP32-FFMA core runs the same cases as a cross-check.
(2) the whole learner step with math_mode=2 against the float64 oracle, same 1e-4 bar as the FFMA path."""
import ctypes as C

import numpy as np
import pytest

import parity

pytestmark = pytest.mark.gpu


def _gemm(native, core, bn, a_km, b_km, M, N, K, splits, seed=0):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((M, K)).astype(np.float32)
    Bm = rng.standard_normal((K, N)).astype(np.float32)
    a_in = np.ascontiguousarray(A if a_km else A.T)            # [M,K] or [K,M]
    b_in = np.ascontiguousarray(Bm.T if b_km else Bm)          # [N,K] or [K,N]
    out = np.zeros((splits, M + 1, N), np.float32)
    native.check(native.lib.drl_debug_gemm(core, bn, int(a_km), int(b_km), M, N, K, splits,
                                           native.ptr(a_in), native.ptr(b_in), native.ptr(out)))
    ref = A.astype(np.float64) @ Bm.astype(np.float64)
    got = out[:, :M].astype(np.float64).sum(0)
    err = np.max(np.abs(got - ref)) / np.max(np.abs(ref))
    cs_err = None
    if not b_km:
        cs = out[:, M].astype(np.float64).sum(0)
        cs_ref = Bm.astype(np.float64).sum(0)
        cs_err = np.max(np.abs(cs - cs_ref)) / np.max(np.abs(cs_ref))
    return err, cs_err


@pytest.mark.parametrize("a_km,b_km", [(1, 0), (1, 1), (0, 0), (0, 1)])
@pytest.mark.parametrize("bn", [32, 64, 128, 256])
def test_umma_gemm_operand_majors(native, a_km, b_km, bn):
    err, cs = _gemm(native, 2, bn, a_km, b_km, 256, 128, 96, 1)
    assert err < 1e-5, (a_km, b_km, bn, err)
    if cs is not None:
        assert cs < 1e-5, cs


@pytest.mark.parametrize("M,N,K,splits,bn", [(128, 32, 32, 1, 32), (132, 36, 100, 1, 64), (640, 1024, 3648, 4, 128),
                                             (3648, 1024, 576, 1, 256), (640, 1024, 3648, 7, 256), (52, 64, 4096, 7, 64), (1000, 200, 68, 2, 128)])
@pytest.mark.parametrize("a_km,b_km", [(1, 0), (0, 0), (1, 1)])
def test_umma_gemm_shapes_and_splitk(native, M, N, K, splits, bn, a_km, b_km):
    err, cs = _gemm(native, 2, bn, a_km, b_km, M, N, K, splits, seed=M + N)
    assert err < 2e-5, (M, N, K, splits, bn, a_km, b_km, err)
    if cs is not None:
        assert cs < 2e-5, cs


def test_ffma_gemm_cross_check(native):
    for a_km, b_km in ((1, 0), (1, 1), (0, 0), (0, 1)):
        err, cs = _gemm(native, 1, 64, a_km, b_km, 132, 36, 100, 2)
        assert err < 1e-5 and (cs is None or cs < 1e-5)


def _assert_all(errs):
    bad = parity.failures(errs)
    assert not bad, "parity failures (rel err): %s" % sorted(bad.items(), key=lambda kv: -kv[1])[:12]


def test_step_small_config_tensor_core_path(native):
    _assert_all(parity.compare_step(4, T=20, math_mode=2))


def test_step_ffma_path(native):
    """math_mode=1 (FP32 FFMA contractions) stays covered now that the tensor-core path is the default."""
    _assert_all(parity.compare_step(4, T=20, math_mode=1))
    _assert_all(parity.compare_step(32, T=20, layers=False, math_mode=1))


def test_step_reference_config_tensor_core_path(native):
    _assert_all(parity.compare_step(32, T=20, layers=False, math_mode=2))


@pytest.mark.parametrize("B,T,A", [(1, 3, 2), (3, 7, 6), (5, 32, 18)])
def test_step_ragged_shapes_tensor_core_path(native, B, T, A):
    _assert_all(parity.compare_step(B, T=T, A=A, math_mode=2))


def test_two_steps_cuda_graph_tensor_core_path(native):
    _assert_all(parity.compare_step(4, T=20, steps=2, layers=False, use_cuda_graph=True, math_mode=2))


@pytest.mark.parametrize("B,T,A,kw", [(4, 20, 18, {}), (32, 20, 18, {"layers": False}), (5, 32, 18, {}), (1, 3, 2, {}),
                                      (4, 20, 18, {"layers": False, "steps": 2, "use_cuda_graph": True})])
def test_step_persistent_tensor_core_kernels(native, B, T, A, kw):
    """math_mode=3: the persistent, warp-specialised wgmma kernels (the epilogue of one tile overlaps the
    gathers of the next) reach the same 1e-4 bar."""
    _assert_all(parity.compare_step(B, T=T, A=A, math_mode=3, **kw))

