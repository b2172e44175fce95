"""Case table of the element-wise one-launch eval block tests (test_block_eval_fp64_gpu.py) and a
Python restatement of the tile plan in csrc/block_eval.cuh (block_eval_launch_impl: which
EvGeom<K, S, TOH, TOW, TI, CPT> and expansion variant a call gets, and how many tiles it walks).
Plain Python: the CPU suite imports it to check, without a GPU, that the GPU table launches every
compiled kernel."""
import os
import re
from collections import namedtuple

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    "yet_another_mobilenet_series_b200", "csrc")
BLOCK_EVAL_SOURCE = os.path.join(CSRC, "block_eval.cuh")

# One resident CTA per SM on a 132-SM H100 SXM.  A walk case has at least two tiles per CTA of the
# unsplit launch, hence more than one tile per cluster at any cluster size.
H100_SMS = 132
WALK_TILES = 2 * H100_SMS
CLUSTER_SIZES = (2, 4, 8)
KPROJ_COLS = 160          # 16 * kMaxProjChunks: wider outputs take one 7x7 image per tile

# act codes (include/yamb200.h): none, ReLU and ReLU6 run the lean kernels (a clamp of the bf16
# pair), Swish and h-swish the generic ones
LEAN_ACTS = (0, 1, 2)

Geom = namedtuple("Geom", "k s toh tow ti cpt")


def compiled_instantiations(path=None):
    """(Geom, expand) of every launch_eval<EvGeom<...>, expand, CLUSTER> call with literal
    arguments in the block eval header."""
    with open(path or BLOCK_EVAL_SOURCE) as f:
        src = f.read()
    pat = (r"launch_eval<EvGeom<\s*(\d+)\s*,\s*(\d+)\s*,\s*(\d+)\s*,\s*(\d+)\s*,\s*(\d+)\s*,"
           r"\s*(\d+)\s*>\s*,\s*(true|false)\s*,")
    return sorted({(Geom(*map(int, m[:6])), m[6] == "true") for m in re.findall(pat, src)})


def _cdiv(a, b):
    return (a + b - 1) // b


def out_size(n, s):
    return (n - 1) // s + 1


def tiles(geom, N, Ho, Wo):
    return _cdiv(Ho, geom.toh) * _cdiv(Wo, geom.tow) * _cdiv(N, geom.ti)


def plan(N, H, W, Cout, k, s, expand):
    """(Geom, expand, num_tiles) the launcher picks."""
    Ho, Wo = out_size(H, s), out_size(W, s)
    wide = _cdiv(Cout, 16) * 16 > KPROJ_COLS
    cpt = 4
    if k == 3 and s == 2:
        g = Geom(3, 2, 7, 7, 1, 2)
    elif k == 5 and s == 2:
        g = Geom(5, 2, 6, 7, 1, 2)
    elif k == 7:
        g = Geom(7, 2, 4, 7, 1, 2) if s == 2 else Geom(7, 1, 7, 7, 1, 2)
    elif wide:
        g = Geom(k, 1, 7, 7, 1, cpt)
    else:
        g16, g77 = Geom(k, 1, 7, 16, 1, cpt), Geom(k, 1, 7, 7, 2, cpt)
        g = g16 if tiles(g16, N, Ho, Wo) <= tiles(g77, N, Ho, Wo) else g77
    return g, expand, tiles(g, N, Ho, Wo)


# N, H, W, Cin, Chid, Cout, k, s, expand, act, residual, affine (gamma / beta given, else NULL),
# cs (the cluster size of the split runs)
Case = namedtuple("Case", "name N H W Cin Chid Cout k s expand act residual affine cs")

CASES = [
    # k3 stride 2
    Case("k3s2_walk", 11, 57, 57, 16, 96, 24, 3, 2, True, 2, False, True, 2),
    Case("k3s2_odd", 2, 17, 23, 24, 144, 40, 3, 2, True, 3, False, False, 4),
    Case("k3s2_one_pixel", 1, 1, 1, 8, 8, 8, 3, 2, True, 0, False, True, 8),
    Case("k3s2_noexp_walk", 11, 57, 57, 32, 32, 16, 3, 2, False, 1, False, True, 2),
    Case("k3s2_noexp_k256", 2, 29, 29, 256, 256, 24, 3, 2, False, 4, False, True, 4),
    # k3 stride 1, wide outputs: one 7x7 image per tile
    Case("k3_wide_walk", 30, 15, 15, 16, 64, 168, 3, 1, True, 1, False, True, 4),
    Case("k3_wide_1152", 2, 7, 7, 256, 1152, 320, 3, 1, True, 3, False, True, 8),
    Case("k3_wide_noexp_walk", 30, 15, 15, 24, 24, 168, 3, 1, False, 2, False, False, 2),
    Case("k3_wide_noexp_k256", 2, 9, 9, 256, 256, 320, 3, 1, False, 4, False, True, 8),
    # k3 stride 1, 7x16
    Case("k3_7x16_walk", 9, 50, 50, 24, 144, 24, 3, 1, True, 1, True, True, 2),
    Case("k3_7x16_hswish", 2, 28, 28, 32, 192, 32, 3, 1, True, 4, True, False, 4),
    Case("k3_7x16_smallest", 1, 3, 3, 8, 8, 8, 3, 1, True, 0, True, True, 8),
    Case("k3_7x16_noexp_walk", 9, 50, 50, 32, 32, 16, 3, 1, False, 1, False, True, 2),
    Case("k3_7x16_noexp_swish", 2, 28, 28, 96, 96, 96, 3, 1, False, 3, True, True, 2),
    # k3 stride 1, two 7x7 images per tile (odd N: the second image of the last tile is past N)
    Case("k3_7x7x2_walk", 529, 7, 7, 16, 64, 16, 3, 1, True, 2, True, True, 8),
    Case("k3_7x7x2_swish", 5, 7, 7, 160, 960, 160, 3, 1, True, 3, True, True, 8),
    Case("k3_7x7x2_noexp_walk", 529, 7, 7, 16, 16, 24, 3, 1, False, 0, False, True, 2),
    Case("k3_7x7x2_noexp_hswish", 3, 7, 7, 144, 144, 144, 3, 1, False, 4, True, False, 4),
    # k5
    Case("k5s2_walk", 30, 31, 31, 16, 48, 32, 5, 2, True, 2, False, True, 2),
    Case("k5s2_swish", 2, 19, 11, 24, 72, 24, 5, 2, True, 3, False, True, 4),
    Case("k5_wide_walk", 30, 15, 15, 16, 64, 168, 5, 1, True, 1, False, False, 2),
    Case("k5_wide_hswish", 2, 7, 7, 96, 576, 320, 5, 1, True, 4, False, True, 8),
    Case("k5_7x16_walk", 9, 50, 50, 40, 120, 40, 5, 1, True, 2, True, True, 2),
    Case("k5_7x16_swish", 2, 28, 28, 80, 240, 80, 5, 1, True, 3, True, True, 4),
    Case("k5_7x7x2_walk", 529, 7, 7, 16, 48, 16, 5, 1, True, 1, False, True, 2),
    Case("k5_7x7x2_hswish", 5, 7, 7, 96, 288, 96, 5, 1, True, 4, True, False, 4),
    # k7
    Case("k7s2_walk", 22, 29, 29, 16, 64, 24, 7, 2, True, 2, False, True, 2),
    Case("k7s2_swish", 2, 28, 28, 32, 96, 40, 7, 2, True, 3, False, True, 4),
    Case("k7_walk", 30, 15, 15, 16, 64, 16, 7, 1, True, 1, True, True, 2),
    Case("k7_1152", 2, 19, 11, 128, 1152, 192, 7, 1, True, 4, False, True, 8),
]
BY_NAME = {c.name: c for c in CASES}


def case_plan(c):
    return plan(c.N, c.H, c.W, c.Cout, c.k, c.s, c.expand)


def lean(c):
    return c.act in LEAN_ACTS


def slices(c):
    return _cdiv(c.Chid, 64)
