"""Shape table of the depthwise kernel tests and a Python restatement of the host dispatch in
csrc/depthwise.cu (which instantiation and how many tiles a call gets).  Plain Python: the CPU
suite imports it to check, without a GPU, that the GPU table launches every compiled kernel."""
import os
import re
from collections import namedtuple

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    "yet_another_mobilenet_series_b200", "csrc")
DW_SOURCES = [os.path.join(CSRC, "depthwise.cu"), os.path.join(CSRC, "depthwise_narrow.cu")]

# yamb_max_ctas() of a 132-SM H100 SXM (4 CTAs per SM): the largest grid a depthwise launch gets.
# A "walk" case has at least two tiles per CTA, so decode / advance, the cp.async prefetch of the
# next tile, the register-resident statistics and the per-CTA weight-gradient slab all run over
# more than one tile.  The GPU test re-checks against the live yamb_max_ctas().
H100_MAX_CTAS = 4 * 132


def pick_ct(C, rows):
    """Channels per tile; the forward passes Ho as `rows`, the backward H (pick_ct in
    depthwise.cu)."""
    if C <= 8 and rows >= 28:
        return 8
    if C <= 16 and rows >= 14:
        return 16
    if C <= 32:
        return 32
    pad64, pad32 = (C + 63) // 64 * 64, (C + 31) // 32 * 32
    return 32 if pad32 < pad64 else 64


def out_size(n, k, s):
    p = (k - 1) // 2
    return (n + 2 * p - k) // s + 1


def _cdiv(a, b):
    return (a + b - 1) // b


FwdPlan = namedtuple("FwdPlan", "inst ct tw tile_h tile_w tiles_h tiles_w chunks num_tiles")
BwdPlan = namedtuple("BwdPlan", "inst ct tile_h tile_w tiles_h tiles_w chunks num_tiles")


def fwd_plan(N, H, W, C, k, s):
    """dw_fwd_launch: instantiation (k, stride, ct, tw) and output-space tiling."""
    Ho, Wo = out_size(H, k, s), out_size(W, k, s)
    ct = pick_ct(C, Ho)
    tw = 1 if (k == 7 or Wo <= 8) else 2
    toh, tow = 512 // ct, 8 * tw
    th, tws, chunks = _cdiv(Ho, toh), _cdiv(Wo, tow), _cdiv(C, ct)
    return FwdPlan((k, s, ct, tw), ct, tw, toh, tow, th, tws, chunks, chunks * N * th * tws)


def bwd_plan(N, H, W, C, k, s):
    """dw_bwd_launch: instantiation (k, stride, ct) and input-space tiling."""
    ct = pick_ct(C, H)
    tih, tiw = 512 // ct, 8
    th, tws, chunks = _cdiv(H, tih), _cdiv(W, tiw), _cdiv(C, ct)
    return BwdPlan((k, s, ct), ct, tih, tiw, th, tws, chunks, chunks * N * th * tws)


def is_walk(plan, max_ctas=H100_MAX_CTAS):
    return plan.num_tiles >= 2 * max_ctas


def partial_tiles(plan, rows, cols):
    """Whether the last tile row and the last tile column are both cut by the image edge."""
    return rows % plan.tile_h != 0 and cols % plan.tile_w != 0


def compiled_instantiations(paths=None):
    """(forward, backward) instantiation tuples compiled by the depthwise sources: every
    YAMB_FWD_CASE(k, s, ct, tw) and YAMB_DW_BWD(k, s, ct, ...) with literal arguments (the macro
    definitions themselves take parameter names and do not match)."""
    fwd, bwd = [], []
    for path in paths or DW_SOURCES:
        with open(path) as f:
            src = f.read()
        fwd += [tuple(map(int, m)) for m in
                re.findall(r"YAMB_FWD_CASE\(\s*(\d+)\s*,\s*(\d+)\s*,\s*(\d+)\s*,\s*(\d+)\s*\)", src)]
        bwd += [tuple(map(int, m)) for m in
                re.findall(r"YAMB_DW_BWD\(\s*(\d+)\s*,\s*(\d+)\s*,\s*(\d+)\s*,", src)]
    return fwd, bwd


# The original direct cases (small shapes: at most one tile per CTA).
# N, H, W, Ctot, c0, C, k, stride, act, prologue
CASES = [
    (2, 14, 14, 96, 0, 96, 3, 1, 1, True),
    (3, 15, 13, 144, 0, 144, 3, 2, 2, True),
    (2, 12, 12, 64, 16, 32, 5, 1, 3, True),
    (2, 12, 12, 64, 32, 32, 7, 2, 3, True),
    (2, 9, 9, 32, 0, 32, 3, 1, 0, False),
    (1, 7, 7, 960, 0, 960, 3, 1, 1, True),
    (2, 16, 16, 48, 8, 40, 5, 2, 4, True),
    # narrow branches of searched networks: 8- / 16-channel tiles (csrc/depthwise_narrow.cu) are
    # selected for C <= 8 with >= 28 rows and C <= 16 with >= 14 rows
    (2, 56, 56, 40, 24, 8, 3, 1, 3, True),       # AtomNAS block 3: 24 | 8 | 8 channels at 56 x 56
    (2, 56, 56, 40, 32, 8, 7, 1, 3, True),
    (2, 57, 59, 24, 0, 8, 5, 2, 1, True),        # odd sizes, stride 2
    (3, 30, 29, 56, 16, 16, 3, 2, 2, True),      # 16-channel tiles
    (2, 28, 28, 56, 40, 16, 5, 1, 3, True),
    (2, 33, 31, 16, 0, 16, 7, 2, 3, True),
    (2, 64, 64, 8, 0, 8, 3, 1, 0, False),        # no prologue
]

# Walk cases: every compiled instantiation at >= 2 tiles per CTA with partial last tiles.
#   act: 0 none, 1 ReLU, 2 ReLU6, 3 Swish, 4 h-swish (the prologue's activation; ignored without)
#   pro: producer BatchNorm + activation applied on load (else identity input and a residual
#        added to dx in the backward)
#   mom: running-statistics update, momentum (-1 = cumulative) from num_batches_tracked = 5
WalkCase = namedtuple("WalkCase", "N H W ldc c0 C k s act pro mom")
WALK_CASES = [
    WalkCase(264, 65, 17, 8, 0, 8, 3, 1, 0, True, 0.1),  # fwd 3,1,8,2  bwd 3,1,8
    WalkCase(264, 33, 17, 16, 0, 16, 3, 1, 1, True, -1.0),  # fwd 3,1,16,2  bwd 3,1,16
    WalkCase(88, 17, 17, 112, 8, 96, 3, 1, 2, True, 0.1),  # fwd 3,1,32,2  bwd 3,1,32
    WalkCase(132, 9, 17, 128, 0, 128, 3, 1, 3, False, -1.0),  # fwd 3,1,64,2  bwd 3,1,64
    WalkCase(528, 65, 7, 8, 0, 8, 3, 1, 4, True, 0.1),  # fwd 3,1,8,1  bwd 3,1,8
    WalkCase(528, 33, 7, 16, 0, 16, 3, 1, 0, True, -1.0),  # fwd 3,1,16,1  bwd 3,1,16
    WalkCase(176, 17, 7, 96, 0, 96, 3, 1, 1, True, 0.1),  # fwd 3,1,32,1  bwd 3,1,32
    WalkCase(264, 9, 7, 144, 8, 128, 3, 1, 2, False, -1.0),  # fwd 3,1,64,1  bwd 3,1,64
    WalkCase(528, 129, 9, 8, 0, 8, 3, 2, 3, True, 0.1),  # fwd 3,2,8,1  bwd 3,2,8
    WalkCase(264, 129, 33, 8, 0, 8, 3, 2, 4, True, -1.0),  # fwd 3,2,8,2  bwd 3,2,8
    WalkCase(528, 65, 9, 16, 0, 16, 3, 2, 0, True, 0.1),  # fwd 3,2,16,1  bwd 3,2,16
    WalkCase(264, 65, 33, 16, 0, 16, 3, 2, 1, False, -1.0),  # fwd 3,2,16,2  bwd 3,2,16
    WalkCase(176, 33, 9, 112, 8, 96, 3, 2, 2, True, 0.1),  # fwd 3,2,32,1  bwd 3,2,32
    WalkCase(88, 33, 33, 96, 0, 96, 3, 2, 3, True, -1.0),  # fwd 3,2,32,2  bwd 3,2,32
    WalkCase(264, 17, 9, 128, 0, 128, 3, 2, 4, True, 0.1),  # fwd 3,2,64,1  bwd 3,2,64
    WalkCase(132, 17, 33, 128, 0, 128, 3, 2, 0, False, -1.0),  # fwd 3,2,64,2  bwd 3,2,64
    WalkCase(264, 65, 17, 8, 0, 8, 5, 1, 1, True, 0.1),  # fwd 5,1,8,2  bwd 5,1,8
    WalkCase(264, 33, 17, 32, 8, 16, 5, 1, 2, True, -1.0),  # fwd 5,1,16,2  bwd 5,1,16
    WalkCase(88, 17, 17, 96, 0, 96, 5, 1, 3, True, 0.1),  # fwd 5,1,32,2  bwd 5,1,32
    WalkCase(132, 9, 17, 128, 0, 128, 5, 1, 4, False, -1.0),  # fwd 5,1,64,2  bwd 5,1,64
    WalkCase(528, 65, 7, 8, 0, 8, 5, 1, 0, True, 0.1),  # fwd 5,1,8,1  bwd 5,1,8
    WalkCase(528, 33, 7, 16, 0, 16, 5, 1, 1, True, -1.0),  # fwd 5,1,16,1  bwd 5,1,16
    WalkCase(176, 17, 7, 112, 8, 96, 5, 1, 2, True, 0.1),  # fwd 5,1,32,1  bwd 5,1,32
    WalkCase(264, 9, 7, 128, 0, 128, 5, 1, 3, False, -1.0),  # fwd 5,1,64,1  bwd 5,1,64
    WalkCase(528, 129, 9, 8, 0, 8, 5, 2, 4, True, 0.1),  # fwd 5,2,8,1  bwd 5,2,8
    WalkCase(264, 129, 33, 8, 0, 8, 5, 2, 0, True, -1.0),  # fwd 5,2,8,2  bwd 5,2,8
    WalkCase(528, 65, 9, 16, 0, 16, 5, 2, 1, True, 0.1),  # fwd 5,2,16,1  bwd 5,2,16
    WalkCase(264, 65, 33, 16, 0, 16, 5, 2, 2, False, -1.0),  # fwd 5,2,16,2  bwd 5,2,16
    WalkCase(176, 33, 9, 96, 0, 96, 5, 2, 3, True, 0.1),  # fwd 5,2,32,1  bwd 5,2,32
    WalkCase(88, 33, 33, 96, 0, 96, 5, 2, 4, True, -1.0),  # fwd 5,2,32,2  bwd 5,2,32
    WalkCase(264, 17, 9, 128, 0, 128, 5, 2, 0, True, 0.1),  # fwd 5,2,64,1  bwd 5,2,64
    WalkCase(132, 17, 33, 128, 0, 128, 5, 2, 1, False, -1.0),  # fwd 5,2,64,2  bwd 5,2,64
    WalkCase(264, 65, 9, 24, 8, 8, 7, 1, 2, True, 0.1),  # fwd 7,1,8,1  bwd 7,1,8
    WalkCase(264, 33, 9, 16, 0, 16, 7, 1, 3, True, -1.0),  # fwd 7,1,16,1  bwd 7,1,16
    WalkCase(88, 17, 9, 96, 0, 96, 7, 1, 4, True, 0.1),  # fwd 7,1,32,1  bwd 7,1,32
    WalkCase(132, 9, 9, 128, 0, 128, 7, 1, 0, False, -1.0),  # fwd 7,1,64,1  bwd 7,1,64
    WalkCase(264, 129, 17, 8, 0, 8, 7, 2, 1, True, 0.1),  # fwd 7,2,8,1  bwd 7,2,8
    WalkCase(264, 65, 17, 32, 8, 16, 7, 2, 2, True, -1.0),  # fwd 7,2,16,1  bwd 7,2,16
    WalkCase(88, 33, 17, 96, 0, 96, 7, 2, 3, True, 0.1),  # fwd 7,2,32,1  bwd 7,2,32
    WalkCase(132, 17, 17, 128, 0, 128, 7, 2, 4, False, -1.0),  # fwd 7,2,64,1  bwd 7,2,64
]
