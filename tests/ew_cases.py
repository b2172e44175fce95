"""Shape tables of the per-channel kernel tests (tests/test_bn_elementwise_gpu.py) and a Python
restatement of the grid rules of their launchers in csrc/elementwise.cu.  Plain Python: the CPU
suite checks, without a GPU, that every table still reaches the grid path it exists for; the GPU
test re-checks each case against the live SM count.

Grid rules (SMS = multiprocessor count, CG = C / 8 channel groups of 8 channels):
  bn_apply      one thread per (row, channel group), 256 threads per CTA, at most 16 * SMS CTAs;
                the thread walks i += stride (stride = grid * 256) and steps (row, group) forward
                by (stride / CG, stride % CG), wrapping the group past CG
  bn_stats      PX = max(256 // CG, 1) pixel lanes per CTA, grid = min(ceil(M / PX), 4 * SMS);
  bn_reduce     the same with at most 2 * SMS CTAs;
  bn_bwd_apply  grid = min(ceil(M / (4 * PX)), 8 * SMS).  These three read rows
                row, row + rstep, row + 2 rstep, row + 3 rstep (rstep = grid * PX) per iteration,
                guarded by r2 < M, and step row by 4 * rstep
  se_bwd_apply  grid = min(ceil(M / PX), 2 * SMS), one row per iteration, row += grid * PX
  all but bn_apply: 256 % CG != 0 leaves lanes px >= PX idle; CG > 256 takes ceil(CG / 256)
                passes (cgb) over the channel groups, the last one CG % 256 groups wide
  se_pool, se_bwd_reduce: channels in launches of at most 2048; se_chunks pixel chunks per
                sample, taken from the widest launch: min(ceil(4 * SMS / N), max(HW // (4 PX), 1));
                a chunk of ceil(HW / chunks) rows is walked by PX lanes, 4 rows per iteration
                then one at a time; more than one chunk sums per-chunk slabs with det_reduce
  bn_stats, bn_reduce, se_bwd_apply: 2 * C doubles of dynamic shared memory besides the static
                17,424 B, so C >= 1984 needs the launcher's opt-in past the 48 KiB default"""
from collections import namedtuple

H100_SMS = 132


def cdiv(a, b):
    return (a + b - 1) // b


def px_of(C):
    return max(256 // (C // 8), 1)


def cg_passes(C):
    return cdiv(C // 8, 256)


# ---- grid restatements ---------------------------------------------------------------------------
ApplyPlan = namedtuple("ApplyPlan", "grid stride passes wrap")
RowPlan = namedtuple("RowPlan", "px grid rstep iters partial idle_lanes cg_passes")


def apply_plan(M, C, sms):
    total = M * (C // 8)
    grid = min(cdiv(total, 256), 16 * sms)
    stride = grid * 256
    return ApplyPlan(grid, stride, cdiv(total, stride), stride % (C // 8) != 0)


def _rows(M, C, grid, batch):
    px = px_of(C)
    rstep = grid * px
    step = batch * rstep
    return RowPlan(px, grid, rstep, cdiv(M, step), M % step != 0 and batch == 4,
                   (C // 8) <= 256 and 256 % (C // 8) != 0, cg_passes(C))


def stats_plan(M, C, sms):
    return _rows(M, C, min(cdiv(M, px_of(C)), 4 * sms), 4)


def reduce_plan(M, C, sms):
    return _rows(M, C, min(cdiv(M, px_of(C)), 2 * sms), 4)


def bwd_apply_plan(M, C, sms):
    return _rows(M, C, min(cdiv(M, 4 * px_of(C)), 8 * sms), 4)


def se_apply_plan(M, C, sms):
    return _rows(M, C, min(cdiv(M, px_of(C)), 2 * sms), 1)


def se_chunks(N, HW, C, sms):
    """Pixel chunks per sample of se_pool / se_bwd_reduce (from the widest 2048-channel launch)."""
    px = px_of(min(C, 2048))
    want = cdiv(4 * sms, N)
    most = max(HW // (4 * px), 1)
    return max(min(want, most), 1)


def se_lane_iters(N, HW, C, sms):
    """4-row iterations of one pixel lane in the first chunk."""
    rows_per = cdiv(HW, se_chunks(N, HW, C, sms))
    return rows_per // (4 * px_of(min(C, 2048)))


SMEM_STATIC = 17424          # ptxas: cta_stats_merge's red[256][17] floats + arrive_last's flag


def needs_optin(C):
    return SMEM_STATIC + 16 * C > 48 * 1024


# ---- case tables ---------------------------------------------------------------------------------
# act: 0 none, 1 ReLU, 2 ReLU6, 3 Swish, 4 h-swish.  ld > C with c0 > 0 is a channel slice of a
# wider buffer.  `why` names the path the case exists for; check_tables asserts it.

# bn_apply: gate (SE, rows_per_sample rows per sample), residual, residual2
ApplyCase = namedtuple("ApplyCase", "M C ld c0 act gate res res2 why")
APPLY_CASES = [
    ApplyCase(1, 8, 8, 0, 1, 0, False, False, "M=1"),
    ApplyCase(200, 8, 24, 8, 2, 0, True, False, "CG=1"),
    ApplyCase(120000, 40, 40, 0, 0, 0, True, True, "wrap"),
    ApplyCase(30000, 200, 216, 8, 2, 0, False, False, "wrap"),
    ApplyCase(4000, 1280, 1280, 0, 3, 49, True, False, "wrap"),
    ApplyCase(190000, 24, 32, 0, 4, 0, False, True, "passes"),
    ApplyCase(300, 2056, 2064, 8, 1, 100, False, False, "wide"),
    ApplyCase(1030, 64, 64, 0, 2, 7, True, True, "gate"),
]

# bn_stats (forward statistics + nn.BatchNorm2d bookkeeping).  mom: momentum, None = cumulative
# average; affine: gamma / beta given (else NULL); data: "randn" or "shifted" (mean ~20 x std)
StatsCase = namedtuple("StatsCase", "M C ld c0 mom affine data why")
STATS_CASES = [
    StatsCase(200, 8, 8, 0, 0.1, True, "randn", "CG=1"),
    StatsCase(33, 24, 40, 8, 0.01, False, "randn", "idle"),
    StatsCase(600000, 40, 40, 0, None, True, "randn", "passes"),
    StatsCase(90000, 200, 200, 0, 0.1, True, "randn", "idle"),
    StatsCase(5000, 1976, 1976, 0, 0.01, True, "randn", "no-optin"),
    StatsCase(3000, 1984, 1992, 8, 0.1, True, "randn", "optin"),
    StatsCase(3000, 2048, 2048, 0, None, False, "randn", "optin"),
    StatsCase(2000, 2056, 2056, 0, 0.1, True, "randn", "cgb"),
    StatsCase(1500, 2560, 2560, 0, 0.01, True, "randn", "cgb"),
    StatsCase(200000, 64, 64, 0, 0.1, True, "shifted", "shifted"),
    StatsCase(256 * 112 * 112, 32, 32, 0, 0.01, True, "randn", "stem"),
]

# bn_reduce and bn_bwd_apply (the backward pair of a stand-alone BatchNorm, optional activation
# after it: z = z_scale * h + z_shift); use_batch_stats 0 = eval-mode BatchNorm
BwdCase = namedtuple("BwdCase", "M C ld c0 act affine why")
BWD_CASES = [
    BwdCase(1, 8, 8, 0, 1, True, "M=1"),             # bn_bwd_apply only
    BwdCase(200, 8, 16, 8, 2, True, "CG=1"),
    BwdCase(77, 24, 24, 0, 0, False, "idle"),
    BwdCase(300000, 40, 48, 8, 3, True, "passes"),
    BwdCase(60000, 200, 200, 0, 4, True, "idle"),
    BwdCase(150001, 64, 64, 0, 1, True, "passes"),
    BwdCase(3000, 1976, 1976, 0, 2, True, "no-optin"),
    BwdCase(2000, 1984, 1984, 0, 1, True, "optin"),
    BwdCase(2000, 2048, 2056, 8, 0, True, "optin"),
    BwdCase(1500, 2056, 2056, 0, 3, True, "cgb"),
    BwdCase(1200, 2560, 2560, 0, 1, False, "cgb"),
]

# se_pool + se_bwd_reduce: N samples of HW pixels
SeCase = namedtuple("SeCase", "N HW C ld c0 act why")
SE_CASES = [
    SeCase(4, 1, 64, 64, 0, 1, "HW=1"),
    SeCase(3, 7, 24, 40, 8, 3, "HW=7"),
    SeCase(2, 3136, 96, 96, 0, 4, "chunks>1"),
    SeCase(1, 3136, 32, 32, 0, 2, "chunks>1"),
    SeCase(176, 3136, 16, 24, 8, 0, "walk"),
    SeCase(600, 49, 200, 200, 0, 3, "chunks=1"),
    SeCase(2, 49, 2056, 2072, 8, 1, "C>2048"),
    SeCase(3, 784, 2560, 2560, 0, 4, "C>2048"),
]

# se_bwd_apply on a channel slice [c0, c0 + C) of Chid channels: dy / h / dz / gate / dpool all
# with pitch Chid; rows_per_sample HW
SeApplyCase = namedtuple("SeApplyCase", "N HW C Chid c0 act why")
SE_APPLY_CASES = [
    SeApplyCase(2, 49, 8, 8, 0, 1, "CG=1"),
    SeApplyCase(128, 196, 40, 120, 40, 4, "slice"),
    SeApplyCase(40, 784, 24, 64, 16, 3, "passes"),
    SeApplyCase(16, 49, 200, 200, 0, 2, "idle"),
    SeApplyCase(8, 49, 1976, 1976, 0, 3, "no-optin"),
    SeApplyCase(4, 49, 1984, 2000, 16, 0, "optin"),
    SeApplyCase(4, 49, 2048, 2048, 0, 4, "optin"),
    SeApplyCase(3, 49, 2056, 2056, 0, 1, "cgb"),
    SeApplyCase(3, 49, 2560, 2568, 8, 3, "cgb"),
]


def se_apply_boundary_inside(case, sms):
    """Whether a thread's rows cross a sample boundary (rows_per_sample = HW)."""
    p = se_apply_plan(case.N * case.HW, case.C, sms)
    step = p.grid * p.px
    return p.iters >= 2 and step % case.HW != 0


def check_tables(sms):
    """Each case reaches the path its `why` names; together they cover every path the module
    docstring lists."""
    for c in APPLY_CASES:
        p = apply_plan(c.M, c.C, sms)
        assert c.C % 8 == 0 and c.ld % 8 == 0 and c.c0 % 8 == 0 and c.c0 + c.C <= c.ld, c
        if c.why == "wrap":
            assert p.passes >= 2 and p.wrap, (c, p)
        if c.why == "passes":
            assert p.passes >= 2, (c, p)
    assert any(c.M == 1 for c in APPLY_CASES) and any(c.C == 8 and c.M < 256 for c in APPLY_CASES)
    assert {c.act for c in APPLY_CASES} == {0, 1, 2, 3, 4}
    assert any(c.gate for c in APPLY_CASES) and any(c.res2 for c in APPLY_CASES)

    for c in STATS_CASES:
        p = stats_plan(c.M, c.C, sms)
        assert c.c0 + c.C <= c.ld and c.M > 1, c
        if c.why == "passes":
            assert p.iters >= 2 and p.partial, (c, p)
        if c.why == "idle":
            assert p.idle_lanes, (c, p)
        if c.why == "no-optin":
            assert not needs_optin(c.C), c
        if c.why == "optin":
            assert needs_optin(c.C) and p.cg_passes == 1, c
        if c.why == "cgb":
            assert p.cg_passes == 2, c
        if c.why == "stem":
            assert p.iters >= 2 and c.M == 256 * 112 * 112 and c.C == 32, (c, p)
    assert {c.mom for c in STATS_CASES} >= {0.1, 0.01, None}
    assert any(not c.affine for c in STATS_CASES)
    assert any(c.data == "shifted" for c in STATS_CASES)
    assert any(c.C == 2056 for c in STATS_CASES)          # the second pass one group wide

    for c in BWD_CASES:
        r, b = reduce_plan(c.M, c.C, sms), bwd_apply_plan(c.M, c.C, sms)
        if c.why == "passes":
            assert r.iters >= 2 and r.partial and b.iters >= 2 and b.partial, (c, r, b)
        if c.why == "idle":
            assert r.idle_lanes, c
        if c.why == "optin":
            assert needs_optin(c.C) and r.cg_passes == 1, c
        if c.why == "cgb":
            assert r.cg_passes == 2, c
    assert {c.act for c in BWD_CASES} == {0, 1, 2, 3, 4}

    for c in SE_CASES:
        ch = se_chunks(c.N, c.HW, c.C, sms)
        if c.why == "chunks>1":
            assert ch > 1, (c, ch)
        if c.why == "walk":
            assert ch > 1 and se_lane_iters(c.N, c.HW, c.C, sms) >= 2, (c, ch)
        if c.why == "chunks=1":
            assert ch == 1, c
        if c.why == "C>2048":
            assert c.C > 2048 and c.C % 2048 >= 8, c
    assert {1, 7, 3136} <= {c.HW for c in SE_CASES}
    assert any(c.C - 2048 == 8 for c in SE_CASES)          # the second launch 8 channels wide

    for c in SE_APPLY_CASES:
        p = se_apply_plan(c.N * c.HW, c.C, sms)
        assert c.c0 + c.C <= c.Chid, c
        if c.why in ("slice", "passes"):
            assert p.iters >= 2 and se_apply_boundary_inside(c, sms), (c, p)
        if c.why == "slice":
            assert c.c0 > 0 and c.Chid > c.c0 + c.C, c
        if c.why == "idle":
            assert p.idle_lanes, c
        if c.why == "optin":
            assert needs_optin(c.C), c
        if c.why == "cgb":
            assert p.cg_passes == 2, c
    assert any(not needs_optin(c.C) and needs_optin(c.C + 8) for c in STATS_CASES)
