"""GPU parity of every gemm_tc_kernel instantiation (block_n x operand majors x epilogue x
transform) on shapes with tails: K % 64 in {16, 24, 40} on the cp.async, register-transform and
TMA-transform (one- and two-source) loader paths, the wgrad pixel tail, MN-major A of <= 64
channels, a last m-block of <= 64 rows (no upper wgmma half) and narrow K (<= 32).

The consumer issues both 64-row halves and four k16 steps for every k-block, so each of these
checks that the loaders store zeros past K and that rows past M never reach the output or the
BatchNorm statistics.  Same machinery as test_gemm_gpu.py (tests/gpu_probe_gemm.py)."""
import pytest

import gpu_probe_gemm

pytestmark = pytest.mark.gpu

M_TAIL = 7 * 128 + 40    # the last m-block has 40 rows: its upper 64-row half is absent

CASES = {
    # forward, K-major A and B: block_n 64 / 32 / 16, plain cp.async loaders
    "fwd64_k80": dict(M=M_TAIL, N=96, K=80, stats=True),
    "fwd64_k24": dict(M=M_TAIL, N=144, K=24, stats=True),
    "fwd32_k104": dict(M=1000, N=24, K=104, stats=True),
    "fwd32_k16": dict(M=M_TAIL, N=32, K=16),
    "fwd16_k88": dict(M=M_TAIL, N=16, K=88, stats=True),
    # forward with the A transform: register path (K < 64), TMA + in-place path (K >= 64)
    "fwd64_x1_reg_k40": dict(M=M_TAIL, N=96, K=40, a_xform=1, act=2, stats=True),
    "fwd64_x1_reg_k24": dict(M=1000, N=144, K=24, a_xform=1, act=1),
    "fwd64_x1_tma_k144": dict(M=M_TAIL, N=96, K=144, a_xform=1, act=3, stats=True),
    "fwd32_x1_tma_k88": dict(M=1000, N=24, K=88, a_xform=1, act=2, stats=True),
    "fwd16_x1_reg_k24": dict(M=M_TAIL, N=16, K=24, a_xform=1, act=4, stats=True),
    "fwd16_x1_tma_k104": dict(M=M_TAIL, N=16, K=104, a_xform=1, act=1),
    # dgrad: MN-major B (+ residual), plain and two-source A transform
    "dgrad_k152_res": dict(M=M_TAIL, N=24, K=152, b_mn=1, residual=True),
    "dgrad_k16": dict(M=M_TAIL, N=160, K=16, b_mn=1),
    "dgrad_x2_tma_k168_res": dict(M=M_TAIL, N=32, K=168, b_mn=1, a_xform=2, residual=True),
    "dgrad_x2_reg_k40": dict(M=1000, N=24, K=40, b_mn=1, a_xform=2),
    # dgrad with the dz epilogue (one instantiation, with and without the A transform)
    "dz_k88_plain": dict(M=M_TAIL, N=144, K=88, b_mn=1, epi=1, act=2),
    "dz_x2_tma_k88": dict(M=M_TAIL, N=144, K=88, b_mn=1, epi=1, act=2, a_xform=2),
    "dz_x2_reg_k24": dict(M=1000, N=96, K=24, b_mn=1, epi=1, act=3, a_xform=2),
    # wgrad: both MN-major, split-K, pixel tail, MN-major A of <= 64 channels
    "wgrad_m40_k5016": dict(M=40, N=96, K=5016, a_mn=1, b_mn=1, epi=2),
    "wgrad_m200_k3024": dict(M=200, N=24, K=3024, a_mn=1, b_mn=1, epi=2),
    "wgrad_x2reg_x1tma_k4056": dict(M=24, N=144, K=4056, a_mn=1, b_mn=1, epi=2, a_xform=2,
                                    b_xform=1, act=2),
    "wgrad_x2tma_k3024": dict(M=144, N=24, K=3024, a_mn=1, b_mn=1, epi=2, a_xform=2),
    "wgrad_x1tma_k2088": dict(M=96, N=576, K=2088, a_mn=1, b_mn=1, epi=2, b_xform=1, act=3),
}


@pytest.mark.parametrize("name", list(CASES))
def test_gemm_tail_case(built_lib, monkeypatch, name):
    monkeypatch.setitem(gpu_probe_gemm.CASES, name, CASES[name])
    assert gpu_probe_gemm.run_case(name) == 0
