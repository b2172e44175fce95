"""Shape tables of the stem convolution, softmax cross entropy and column-sum kernel tests
(test_tail_fp64_gpu.py), and a Python restatement of their host-side launch plans (csrc/stem.cu,
csrc/loss.cu).  Plain Python: the CPU suite imports it to check, without a GPU, that the GPU
tables reach every path of those kernels."""
from collections import namedtuple

H100_SMS = 132
# 256-thread CTAs an SM can hold at most (2048 threads).  The stem grids are one resident wave,
# SMs x CTAs per SM at the kernel's occupancy; nobody pinned that occupancy for the forward, so a
# "walk" case is sized against this ceiling: at least two tiles per CTA at any occupancy.
CTA_CEIL = 8
STEM_TH, STEM_TW = 16, 32             # output tile of both stem kernels
CE_MAX_C = 4096                       # 32 lanes x 128 logits per lane


def cdiv(a, b):
    return (a + b - 1) // b


# ---- stem convolution ------------------------------------------------------------------------------
StemPlan = namedtuple("StemPlan", "Ho Wo tiles_h tiles_w num_tiles aligned")


def stem_plan(N, H, W):
    """stem_fill: output size (3x3, stride 2, pad 1) and the 16 x 32 output tiling; `aligned`: the
    image rows are 4-byte aligned (3W even) and staged with cp.async, else element by element."""
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    th, tw = cdiv(Ho, STEM_TH), cdiv(Wo, STEM_TW)
    return StemPlan(Ho, Wo, th, tw, N * th * tw, (3 * W) % 2 == 0)


def stem_wgrad_slots(grid, Cout):
    """Partial slabs of the weight gradient: grid x PS pixel subsets, PS = 256 / Cout."""
    return grid * (256 // Cout)


def stem_is_walk(plan, sms=H100_SMS):
    return plan.num_tiles >= 2 * CTA_CEIL * sms


def stem_cut_edges(plan):
    """The last tile row and the last tile column are both cut by the image edge."""
    return plan.Ho % STEM_TH != 0 and plan.Wo % STEM_TW != 0


STEM_FWD_COUT = (8, 16, 24, 32, 40, 48, 56, 64)
STEM_WGRAD_COUT = (8, 16, 32, 64)

StemCase = namedtuple("StemCase", "N H W Cout")
# Direct cases: at most a few tiles per CTA.  37 x 37 / 45 x 29: odd widths (2-byte staging), cut
# tiles; 38 x 46 / 66 x 70: even widths (cp.async staging), two tile columns; 1..3 pixel images.
STEM_CASES = [StemCase(3, 37, 37, co) for co in STEM_FWD_COUT] + \
    [StemCase(2, 38, 46, co) for co in STEM_FWD_COUT] + [
    StemCase(2, 45, 29, 16), StemCase(2, 66, 70, 32),
    StemCase(3, 1, 1, 8), StemCase(2, 1, 2, 16), StemCase(2, 2, 1, 64), StemCase(1, 2, 2, 32),
    StemCase(2, 3, 3, 24), StemCase(3, 1, 3, 8), StemCase(1, 3, 2, 56), StemCase(2, 2, 3, 64),
]
# Walks: 2112 tiles = 2 x 8 x 132.  230 x 230 -> 115 x 115 outputs (even width: cp.async), 225 x 225
# -> 113 x 113 (odd width: 2-byte path); both cut their last tile row and column.  224 x 224
# would not do: Ho = 112 fills its last tile row.
STEM_WALK_CASES = [StemCase(66, 230, 230, co) for co in STEM_WGRAD_COUT] + \
    [StemCase(66, 225, 225, co) for co in STEM_WGRAD_COUT]

# eval forward: every activation at these widths (a direct case of each staging path)
STEM_EVAL_COUT = (8, 24, 56, 64)
STEM_EVAL_SHAPES = ((3, 37, 37), (2, 38, 46))


# ---- softmax cross entropy ----------------------------------------------------------------------
def ce_fwd_grid(N):
    """softmax_ce_fwd_launch: one warp per row, 8 rows per CTA."""
    return cdiv(N, 8)


def ce_bwd_grid(N, sms=H100_SMS):
    """softmax_ce_bwd_launch: grid-stride over rows, min(N, 2 x SMs) CTAs."""
    return min(N, 2 * sms)


def pairs_per_thread(C):
    """Column pairs each of the 256 threads covers (backward and column sum)."""
    return cdiv(C // 2, 256)


# ld: logits pitch (POISON between C and ld); ldg: G pitch; ldd: dlogits pitch (SENTINEL in both
# paddings); eps: label smoothing.  Cases with even C and pitches also run the backward.
CeCase = namedtuple("CeCase", "N C ld ldg ldd eps")
CE_CASES = [
    CeCase(7, 1, 3, 2, 2, 0.1),
    CeCase(9, 2, 2, 2, 2, 0.0),
    CeCase(5, 4, 4, 6, 8, 0.1),
    CeCase(13, 5, 7, 5, 5, 0.1),
    CeCase(8, 6, 6, 8, 6, 0.0),
    CeCase(7, 10, 10, 10, 12, 0.1),
    CeCase(33, 31, 35, 31, 31, 0.1),
    CeCase(64, 32, 32, 40, 32, 0.1),
    CeCase(17, 33, 40, 33, 33, 0.0),
    CeCase(70, 64, 66, 64, 72, 0.0),
    CeCase(256, 1000, 1000, 1000, 1000, 0.1),
    CeCase(45, 1001, 1001, 1003, 1001, 0.1),
    CeCase(600, 1000, 1024, 1002, 1008, 0.1),
    CeCase(600, 1000, 1000, 1000, 1000, 0.0),
    CeCase(300, 4096, 4104, 4096, 4100, 0.1),
    CeCase(10, 4096, 4096, 4100, 4096, 0.0),
]


def ce_has_bwd(c):
    return c.C % 2 == 0 and c.ldg % 2 == 0 and c.ldd % 2 == 0


# ---- column sum ---------------------------------------------------------------------------------
def colsum_grid(M, C):
    """colsum_bf16_launch: (column-pair blocks of 256, row slabs min(M, 32))."""
    return (cdiv(C // 2, 256), min(M, 32))


ColsumCase = namedtuple("ColsumCase", "M C ld")
COLSUM_CASES = [ColsumCase(M, C, C + (8 if (M + C // 2) % 2 else 0))
                for M in (1, 31, 32, 33, 4097) for C in (2, 510, 512, 514, 1000, 1280)]
