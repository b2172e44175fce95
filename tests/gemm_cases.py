"""Case table of the pointwise GEMM tests (yamb_pointwise_gemm, csrc/gemm_tc.cu).

Plain data: each case gives the shape, the operand majors, the epilogue, the operand transforms and
activation, the SE gate, the operand pitches and output slice, max_ctas, the BatchNorm options and
a seed.  tests/test_gemm_plan_cpu.py checks, through the library's own plan query
(yamb_gemm_plan), that the table reaches every compiled instantiation and every launch-plan axis;
tests/test_gemm_fp64_gpu.py runs every case against a float64 reference."""
import ctypes as C
import os
import re
from dataclasses import dataclass
from typing import Optional

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GEMM_SOURCE = os.path.join(ROOT, "yet_another_mobilenet_series_b200", "csrc", "gemm_tc.cu")
PLAN_SMS = 132           # the H100 SXM's SM count: the table is laid out for it
MAX_BYTES = 1 << 30      # device memory per case, fp64 reference included
REF_ROWS = 1 << 16       # rows of the fp64 reference formed at a time


@dataclass(frozen=True)
class Case:
    name: str
    M: int
    N: int
    K: int
    a_mn: int = 0
    b_mn: int = 0
    epi: int = 0
    a_xform: int = 0          # 0 none, 1 BN-apply + activation, 2 two-source affine
    b_xform: int = 0
    act: int = 0              # activation of the mode-1 transform, and h_act of epi 1
    gate: int = 0             # SE gate rows_per_sample on the mode-1 operand (0: no gate)
    residual: bool = False
    stats: bool = False       # epi 0: BatchNorm forward statistics
    pad: int = 0              # extra columns in every operand / output pitch (NaN in inputs)
    c0: int = 0               # channel offset of the output (and H / residual) slice
    max_ctas: int = 0
    mom: Optional[float] = 0.01
    affine: bool = True       # gamma / beta (False: NULL)
    running: bool = True      # running statistics and saved mean / invstd (False: NULL)
    use_batch_stats: int = 1  # epi 1
    grads: bool = True        # epi 1: dgamma / dbeta buffers (False: NULL)
    shifted: bool = False     # D's channel means ~8x their std (the long-chain statistics case)
    seed: int = 0
    why: str = ""


M_TAIL = 7 * 128 + 40    # the last m-block has 40 rows: its upper 64-row half is absent


def _old(name, M, N, K, a_mn=0, b_mn=0, epi=0, a_xform=0, b_xform=0, act=0, stats=False,
         residual=False):
    """A case of the earlier rel-L2 tests, under its old name."""
    return Case(name, M, N, K, a_mn=a_mn, b_mn=b_mn, epi=epi, a_xform=a_xform, b_xform=b_xform,
                act=act, stats=stats, residual=residual, why="earlier parity case")


CASES = [
    # ---- the earlier parity cases (forward / dgrad / wgrad, transforms, BN epilogues) ----
    _old("plain_small", 256, 64, 64),
    _old("plain_k16", 384, 96, 16),
    _old("plain_k24_n24", 200, 24, 24),
    _old("plain_k144_n32", 1000, 32, 144),
    _old("plain_multi_n", 640, 320, 960),
    _old("plain_n960", 300, 960, 160),
    _old("plain_big", 128 * 148 * 3 + 40, 96, 16),
    _old("stats", 1000, 144, 24, stats=True),
    _old("stats_multi_n", 5000, 576, 96, stats=True),
    _old("xform1", 1000, 32, 192, a_xform=1, act=1, stats=True),
    _old("xform1_swish", 777, 160, 576, a_xform=1, act=3),
    _old("dgrad", 1000, 144, 24, b_mn=1),
    _old("dgrad_big", 900, 960, 160, b_mn=1),
    _old("residual", 1000, 24, 144, b_mn=1, residual=True),
    _old("wgrad", 96, 16, 5000, a_mn=1, b_mn=1, epi=2),
    _old("wgrad_big", 320, 960, 3000, a_mn=1, b_mn=1, epi=2),
    _old("wgrad_xform", 24, 144, 4000, a_mn=1, b_mn=1, epi=2, b_xform=1, act=2),
    _old("dz", 1000, 144, 24, b_mn=1, epi=1, act=1),
    _old("dz_swish_multi", 700, 576, 96, b_mn=1, epi=1, act=3),
    _old("xform2", 1000, 24, 144, b_mn=1, a_xform=2, residual=True),
    _old("wgrad_xform2", 144, 24, 4000, a_mn=1, b_mn=1, epi=2, a_xform=2),
    # ---- the earlier tail cases: K % 64 tails, last m-block of <= 64 rows, narrow K ----
    _old("fwd64_k80", M_TAIL, 96, 80, stats=True),
    _old("fwd64_k24", M_TAIL, 144, 24, stats=True),
    _old("fwd32_k104", 1000, 24, 104, stats=True),
    _old("fwd32_k16", M_TAIL, 32, 16),
    _old("fwd16_k88", M_TAIL, 16, 88, stats=True),
    _old("fwd64_x1_reg_k40", M_TAIL, 96, 40, a_xform=1, act=2, stats=True),
    _old("fwd64_x1_reg_k24", 1000, 144, 24, a_xform=1, act=1),
    _old("fwd64_x1_tma_k144", M_TAIL, 96, 144, a_xform=1, act=3, stats=True),
    _old("fwd32_x1_tma_k88", 1000, 24, 88, a_xform=1, act=2, stats=True),
    _old("fwd16_x1_reg_k24", M_TAIL, 16, 24, a_xform=1, act=4, stats=True),
    _old("fwd16_x1_tma_k104", M_TAIL, 16, 104, a_xform=1, act=1),
    _old("dgrad_k152_res", M_TAIL, 24, 152, b_mn=1, residual=True),
    _old("dgrad_k16", M_TAIL, 160, 16, b_mn=1),
    _old("dgrad_x2_tma_k168_res", M_TAIL, 32, 168, b_mn=1, a_xform=2, residual=True),
    _old("dgrad_x2_reg_k40", 1000, 24, 40, b_mn=1, a_xform=2),
    _old("dz_k88_plain", M_TAIL, 144, 88, b_mn=1, epi=1, act=2),
    _old("dz_x2_tma_k88", M_TAIL, 144, 88, b_mn=1, epi=1, act=2, a_xform=2),
    _old("dz_x2_reg_k24", 1000, 96, 24, b_mn=1, epi=1, act=3, a_xform=2),
    _old("wgrad_m40_k5016", 40, 96, 5016, a_mn=1, b_mn=1, epi=2),
    _old("wgrad_m200_k3024", 200, 24, 3024, a_mn=1, b_mn=1, epi=2),
    _old("wgrad_x2reg_x1tma_k4056", 24, 144, 4056, a_mn=1, b_mn=1, epi=2, a_xform=2, b_xform=1,
         act=2),
    _old("wgrad_x2tma_k3024", 144, 24, 3024, a_mn=1, b_mn=1, epi=2, a_xform=2),
    _old("wgrad_x1tma_k2088", 96, 576, 2088, a_mn=1, b_mn=1, epi=2, b_xform=1, act=3),

    # ---- SE gates: project forward (K-major A) and project wgrad (MN-major B) ----
    Case("proj_gate_reg_k40", 1000, 24, 40, a_xform=1, act=3, gate=49, stats=True,
         why="a_gate on the register path, samples of 49 rows end inside tiles"),
    Case("proj_gate_tma_k144", M_TAIL, 40, 144, a_xform=1, act=4, gate=196, stats=True,
         why="a_gate on the TMA path, 196-row samples across tile edges"),
    Case("proj_gate_relu6_rps1", 400, 32, 56, a_xform=1, act=2, gate=1,
         why="a_gate with one row per sample (exact operands)"),
    Case("wgrad_gate_reg_n40", 40, 40, 4000, a_mn=1, b_mn=1, epi=2, b_xform=1, act=3, gate=200,
         why="b_gate on the register path (N < 64), 200-row samples vs 64-row k-blocks"),
    Case("wgrad_gate_tma_n96", 24, 96, 3136, a_mn=1, b_mn=1, epi=2, b_xform=1, act=2, gate=196,
         why="b_gate on the TMA path"),
    Case("wgrad_gate_tma_rps1", 16, 64, 1000, a_mn=1, b_mn=1, epi=2, b_xform=1, act=4, gate=1,
         why="b_gate with one row per sample"),
    Case("wgrad_b1_reg_n24", 56, 24, 2504, a_mn=1, b_mn=1, epi=2, b_xform=1, act=1,
         why="B transform through registers (N < 64), no gate"),
    # ---- two-source B (mode 2) on both loader paths ----
    Case("wgrad_b2_reg_n24", 40, 24, 2000, a_mn=1, b_mn=1, epi=2, b_xform=2,
         why="two-source B through registers"),
    Case("wgrad_b2_tma_n96", 40, 96, 2000, a_mn=1, b_mn=1, epi=2, b_xform=2,
         why="two-source B by TMA"),
    # ---- strided operands, channel slices, padding that must not be read ----
    Case("fwd_slice_stats", 1000, 48, 56, stats=True, pad=16, c0=24, max_ctas=5,
         why="pitches > K / N, output slice at channel 24, 8-tile walks"),
    Case("dgrad_slice_res", M_TAIL, 96, 40, b_mn=1, residual=True, pad=8, c0=32,
         why="sliced dgrad with residual, pitches > N"),
    Case("dz_slice_x2", 1000, 72, 88, b_mn=1, epi=1, act=4, a_xform=2, pad=24, c0=8,
         why="sliced epi 1 (multi-branch dgrad), ldh / ldd / lda2 > N"),
    Case("wgrad_slice", 48, 56, 3000, a_mn=1, b_mn=1, epi=2, pad=8, c0=16,
         why="epi 2 into a slice of a wider fp32 gradient"),
    # ---- BatchNorm bookkeeping in the epilogues ----
    Case("stats_cumulative", 1500, 40, 72, stats=True, mom=None,
         why="momentum=None: cumulative running statistics"),
    Case("stats_mom01_noaffine", M_TAIL, 64, 16, stats=True, mom=0.1, affine=False,
         why="NULL gamma / beta, momentum 0.1"),
    Case("stats_no_running", 1000, 96, 32, stats=True, running=False,
         why="NULL running statistics and saved mean / invstd"),
    Case("dz_eval_bn", 1000, 64, 48, b_mn=1, epi=1, act=1, use_batch_stats=0,
         why="use_batch_stats = 0: dh = ca * dz"),
    Case("dz_no_grads", 1000, 40, 24, b_mn=1, epi=1, act=2, grads=False, affine=False,
         why="NULL dgamma / dbeta / gamma"),
    # ---- the launch plan ----
    Case("fwd_k8_walk_odd", 23 * 128 - 64, 32, 8, stats=True, max_ctas=5,
         why="K = 8, an odd number of tiles walked by 5 CTAs, register statistics"),
    Case("fwd_k56_walk2", 21 * 128, 64, 56, a_xform=1, act=1, stats=True, max_ctas=2,
         why="K % 64 = 56, many tiles per CTA, warpgroup hand-over"),
    Case("fwd_wg2x_walk", 9 * 128 + 8, 40, 200, a_xform=1, act=4, stats=True, max_ctas=3,
         why="warps 8-11 load (wg2x), one epilogue warpgroup walks every tile"),
    Case("dgrad_res_walk", 11 * 128 + 24, 96, 72, b_mn=1, residual=True, max_ctas=4,
         why="residual rows prefetched for the next tile of the walk"),
    Case("dz_walk_reg_stats", 13 * 128 + 16, 64, 40, b_mn=1, epi=1, act=3, max_ctas=3,
         why="epi 1, single n-block: register statistics over a walk, H rows prefetched"),
    Case("dz_n960_x2", 1200, 960, 144, b_mn=1, epi=1, act=2, a_xform=2,
         why="wide epi 1 with a two-source A: one staging buffer"),
    Case("wgrad_ksplit_uneven", 64, 64, 64 * 37, a_mn=1, b_mn=1, epi=2,
         why="split-K with an uneven last slab"),
    Case("wgrad_ksplit_capped", 64, 64, 64 * 37, a_mn=1, b_mn=1, epi=2, max_ctas=3,
         why="max_ctas small enough to change ksplit"),
    Case("wgrad_k_tail8", 32, 40, 3000 + 8, a_mn=1, b_mn=1, epi=2, a_xform=1, act=1,
         why="MN-major A of <= 64 rows transformed, K % 64 = 8"),
    Case("stats_long_chain", 800000, 64, 32, stats=True, shifted=True, mom=0.1,
         why="~800k rows, channel mean ~8x std: Sum h^2 - M mean^2 cancellation"),
]

BY_NAME = {c.name: c for c in CASES}
assert len(BY_NAME) == len(CASES), "duplicate case names"


# ---- layouts -------------------------------------------------------------------------------------
def pitches(c):
    """Leading dimensions (elements) of A, A2, B, B2, D, H / residual."""
    a_cols = c.M if c.a_mn else c.K
    b_cols = c.N if c.b_mn else c.K
    return dict(lda=a_cols + c.pad, ldb=b_cols + c.pad, ldd=c.c0 + c.N + c.pad,
                lds=c.c0 + c.N + c.pad)


def rows_of(c):
    return (c.K if c.a_mn else c.M), (c.K if c.b_mn else c.N)


def est_bytes(c):
    """Device memory of one case: inputs, outputs (with a second copy for repeat runs) and the
    fp64 reference formed REF_ROWS rows at a time."""
    p = pitches(c)
    ra, rb = rows_of(c)
    n = 2 * (ra + 1) * p["lda"] * (2 if c.a_xform == 2 else 1)
    n += 2 * (rb + 1) * p["ldb"] * (2 if c.b_xform == 2 else 1)
    n += 2 * (c.M + 1) * p["lds"] * (2 if (c.epi == 1 or c.residual) else 0)
    n += 4 * (c.M + 1) * p["ldd"] * 3
    rows = c.M if c.epi == 2 else min(c.M, REF_ROWS)   # epi 0 / 1: formed a row chunk at a time
    n += 8 * (rows * c.K + c.N * c.K) * 4          # fp64 operands, magnitudes and bands
    n += 8 * rows * c.N * 8                        # fp64 reference and its bounds
    return n


def gemm_struct(nat, c, ptrs=None, max_ctas=None):
    """The yamb_gemm of case c.  ptrs: name -> device address (fake addresses for the plan query);
    missing pointers are NULL."""
    ptrs = ptrs or {}
    p = pitches(c)
    g = nat.Gemm()
    g.M, g.N, g.K = c.M, c.N, c.K
    g.a_mn_major, g.b_mn_major = c.a_mn, c.b_mn
    g.A, g.lda = ptrs.get("A"), p["lda"]
    g.B, g.ldb = ptrs.get("B"), p["ldb"]
    g.D, g.ldd = ptrs.get("D"), p["ldd"]
    g.epi = c.epi
    g.a_xform, g.b_xform = c.a_xform, c.b_xform
    g.a_act = c.act if c.a_xform == 1 else 0
    g.b_act = c.act if c.b_xform == 1 else 0
    for s in ("a", "b"):
        for k in ("scale", "shift", "scale2"):
            setattr(g, s + "_" + k, ptrs.get(s + "_" + k))
    g.A2, g.lda2 = ptrs.get("A2"), p["lda"]
    g.B2, g.ldb2 = ptrs.get("B2"), p["ldb"]
    if c.residual:
        g.residual, g.ldr = ptrs.get("residual"), p["lds"]
    if c.epi == 1:
        g.H, g.ldh = ptrs.get("H"), p["lds"]
        g.h_scale, g.h_shift, g.h_act = ptrs.get("h_scale"), ptrs.get("h_shift"), c.act
    if c.gate:
        if c.a_xform == 1:
            g.a_gate = ptrs.get("gate")
        else:
            g.b_gate = ptrs.get("gate")
        g.gate_rows_per_sample = c.gate
    g.max_ctas = c.max_ctas if max_ctas is None else max_ctas
    return g


_FAKE = 1 << 32


def fake_ptrs(c):
    names = ["A", "B", "D", "a_scale", "a_shift", "a_scale2", "b_scale", "b_shift", "b_scale2",
             "A2", "B2", "residual", "H", "h_scale", "h_shift", "gate"]
    return {k: _FAKE + (i << 28) for i, k in enumerate(names)}


def plan(lib, nat, c, sms=PLAN_SMS, max_ctas=None, g=None):
    """The library's plan of case c (yamb_gemm_plan with `sms` SMs): (rc, info)."""
    if g is None:
        g = gemm_struct(nat, c, fake_ptrs(c), max_ctas)
    keep = []
    if c.epi == 0 and c.stats:
        f = nat.BnFwd()
        keep.append(f)
        g.bn_fwd = C.pointer(f)
    if c.epi == 1:
        b = nat.BnBwd()
        keep.append(b)
        g.bn_bwd = C.pointer(b)
    info = nat.GemmPlanInfo()
    rc = lib.yamb_gemm_plan(C.byref(g), sms, C.byref(info))
    return rc, info


def inst_of(info):
    return (info.xf, info.epi, info.block_n, info.a_mn, info.b_mn)


def tiles_per_cta(info):
    return -(-info.num_work // info.grid)


# ---- the instantiations the sources compile ------------------------------------------------------
def compiled_instantiations(path=GEMM_SOURCE):
    """(XF, EP, BN, AMN, BMN) of every launch_tc the host code can select: pick_tc<EP, BN, AMN,
    BMN>(xf) stands for both XF values, launch_tc<XF, EP, BN, AMN, BMN> for itself."""
    src = open(path).read()
    body = src[src.index("static int gemm_plan("):]
    out = set()
    for m in re.finditer(r"pick_tc<\s*(\d+)\s*,\s*(\d+)\s*,\s*(\d+)\s*,\s*(\d+)\s*>\s*\(", body):
        ep, bn, am, bm = (int(v) for v in m.groups())
        out |= {(1, ep, bn, am, bm), (0, ep, bn, am, bm)}
    for m in re.finditer(r"&launch_tc<\s*(true|false)\s*,\s*(\d+)\s*,\s*(\d+)\s*,\s*(\d+)\s*,\s*(\d+)\s*>",
                         body):
        xf = 1 if m.group(1) == "true" else 0
        out.add((xf,) + tuple(int(v) for v in m.groups()[1:]))
    return sorted(out)
