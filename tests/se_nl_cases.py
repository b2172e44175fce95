"""Case tables of the element-wise Squeeze-and-Excitation, non-local and InstanceNorm kernel tests
(test_se_nl_fp64_gpu.py), and a Python restatement of their host-side launch plans (csrc/se_fc.cu,
csrc/nonlocal.cu, csrc/instance_norm.cu) with the SM count as a parameter.  The plan constants are
read out of the sources, so a changed kernel constant fails the CPU test (test_se_nl_plan_cpu.py)
instead of silently moving what the tables reach.  Plain Python: the CPU suite imports it."""
import os
import re
from collections import namedtuple

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    "yet_another_mobilenet_series_b200", "csrc")
SE_SOURCE = os.path.join(CSRC, "se_fc.cu")
NL_SOURCE = os.path.join(CSRC, "nonlocal.cu")
IN_SOURCE = os.path.join(CSRC, "instance_norm.cu")

H100_SMS = 132            # H100 SXM
H100_PCIE_SMS = 114


def cdiv(a, b):
    return (a + b - 1) // b


def _read(path):
    with open(path) as f:
        return f.read()


def _one(pat, src, what):
    m = re.findall(pat, src)
    assert len(m) == 1, "%s: expected one match of %r, found %d" % (what, pat, len(m))
    return m[0]


def parse_constants(se=None, nl=None, inorm=None):
    """The launch-plan constants as the sources state them."""
    se, nl, inorm = _read(se or SE_SOURCE), _read(nl or NL_SOURCE), _read(inorm or IN_SOURCE)
    t, k = _one(r"constexpr int kSgT = (\d+), kSgK = (\d+);", se, "se_fc tile")
    c = {"kSgT": int(t), "kSgK": int(k),
         "se_finish_rows": int(_one(r"nrow = \(a->N \+ \d+\) / (\d+);\n\s*if \(\(rc = det_alloc"
                                    r"\(\(size_t\)nrow \* a->R", se, "finish slab")),
         "se_dt_rows": int(_one(r"se_dt_kernel<<<grid, 256, 0, st>>>\([^;]*colpart, (\d+)\);", se,
                                "dt slab")),
         "se_max_c": int(_one(r"C > (\d+) \|\| R >", se, "C limit")),
         "se_max_r": int(_one(r"R > (\d+) \|\| N >", se, "R limit")),
         "se_max_n_slabs": int(_one(r"N > \d+ \* (\d+)\)", se, "N limit")),
         "gram_rows": int(_one(r"int R = rows < (\d+) \? rows : \d+;", nl, "gram rows")),
         "gram_min_rows": int(_one(r"while \(R > (\d+) && \(long long\)\(\(rows \+ R - 1\) / R\) \* "
                                   r"a->N < 2LL \* max_ctas\(\) &&", nl, "gram halving floor")),
         "gram_slab_mb": int(_one(r"<= \((\d+)LL << 20\)\)", nl, "gram slab cap")),
         "gram_smem_kb": int(_one(r"if \(smem > (\d+) \* 1024\) return set_error\(YAMB_EINVAL, "
                                  r"\"nl_gram", nl, "gram smem")),
         "rowmat_rows": int(_one(r"int R = (\d+);\n\s*while \(R > \d+", nl, "rowmat rows")),
         "rowmat_min_rows": int(_one(r"while \(R > (\d+) && \(long long\)\(\(rows \+ R - 1\) / R\)"
                                     r" \* a->N < 2LL \* max_ctas\(\)\) R /= 2;", nl,
                                     "rowmat halving floor")),
         "rowmat_smem_kb": int(_one(r"if \(smem > (\d+) \* 1024\) return set_error\(YAMB_EINVAL, "
                                    r"\"nl_rowmat", nl, "rowmat smem")),
         "kThreads": int(_one(r"constexpr int kThreads = (\d+);", inorm, "kThreads")),
         "kChunk": int(_one(r"constexpr int kChunk = (\d+);", inorm, "kChunk")),
         "kUnroll": int(_one(r"constexpr int kUnroll = (\d+);", inorm, "kUnroll"))}
    return c


# the mirror below; test_se_nl_plan_cpu.py checks it against parse_constants()
K = {"kSgT": 64, "kSgK": 16, "se_finish_rows": 8, "se_dt_rows": 32, "se_max_c": 4096,
     "se_max_r": 1024, "se_max_n_slabs": 65535, "gram_rows": 64, "gram_min_rows": 16,
     "gram_slab_mb": 16, "gram_smem_kb": 200, "rowmat_rows": 32, "rowmat_min_rows": 8,
     "rowmat_smem_kb": 220, "kThreads": 256, "kChunk": 64, "kUnroll": 4}
SE_MAX_N = K["se_finish_rows"] * K["se_max_n_slabs"]


# ---- Squeeze-and-Excitation ----------------------------------------------------------------------
SplitPlan = namedtuple("SplitPlan", "ksplit k_per_slab nslab tiles")


def se_ksplit(M, N, Kd, sms=H100_SMS):
    """se_ksplit: K slabs wanted for a split-K product [M][N] with K = Kd."""
    T, KC = K["kSgT"], K["kSgK"]
    tiles = cdiv(M, T) * cdiv(N, T)
    want = min(cdiv(2 * sms, tiles), cdiv(Kd, 4 * KC))
    return max(want, 1)


def se_split(Kd, ksplit):
    """se_split: (k_per_slab, slabs written)."""
    kps = cdiv(cdiv(Kd, ksplit), K["kSgK"]) * K["kSgK"]
    return kps, cdiv(Kd, kps)


def se_product_plan(M, N, Kd, sms=H100_SMS):
    """The split-K products u and du ([N][R], K = C)."""
    ks = se_ksplit(M, N, Kd, sms)
    kps, nslab = se_split(Kd, ks)
    return SplitPlan(ks, kps, nslab, cdiv(M, K["kSgT"]) * cdiv(N, K["kSgT"]))


SePlan = namedtuple("SePlan", "split finish_slabs dt_slabs")


def se_plan(N, C, R, sms=H100_SMS):
    return SePlan(se_product_plan(N, R, C, sms), cdiv(N, K["se_finish_rows"]),
                  cdiv(N, K["se_dt_rows"]))


SeCase = namedtuple("SeCase", "name N C R act")
AUTONL_L_SE = ((1152, 48),)                     # (C, R) of AutoNL-L's SE branches
ATOMNAS_CP_SE = ((1390, 96), (2310, 96))        # AtomNAS-C+
SE_CASES = [
    SeCase("tiny", 1, 8, 1, 2),
    SeCase("n7_r2", 7, 72, 2, 0),
    SeCase("n8_r4", 8, 72, 4, 1),
    SeCase("n9_r10", 9, 200, 10, 2),
    SeCase("n31", 31, 136, 10, 3),
    SeCase("n32", 32, 72, 65, 4),
    SeCase("n33", 33, 264, 20, 1),
    SeCase("r65_tiles", 100, 1390, 65, 3),
    SeCase("r1024", 65, 520, 1024, 4),
    SeCase("c4096", 33, 4096, 64, 2),
    SeCase("c64_one_slab", 70, 64, 24, 3),
    SeCase("tiles_one_slab", 1100, 136, 1000, 0),
    SeCase("autonl_l", 256, 1152, 48, 3),
    SeCase("atomnas_cp_1390", 256, 1390, 96, 3),
    SeCase("atomnas_cp_2310", 256, 2310, 96, 1),
    SeCase("n_max", SE_MAX_N, 8, 2, 4),
]
SE_ACT_EDGES = (0.0, -0.0, 6.0, -3.0, 3.0, -100.0, 100.0)   # b_r at the planted rows (pooled = 0)


# ---- non-local gram ------------------------------------------------------------------------------
def sub_size(n, sub):
    return cdiv(n, sub)


GramPlan = namedtuple("GramPlan", "rows R chunks last direct smem")


def gram_plan(N, H, W, sub, I, J, sms=H100_SMS):
    """nl_gram_launch: rows per CTA (halved while the batch cannot fill the SMs and the chunk slabs
    stay under the cap), row chunks, and direct store (one chunk) versus det_reduce."""
    rows = sub_size(H, sub) * sub_size(W, sub)
    n_out = N * I * J
    R = min(rows, K["gram_rows"])
    while (R > K["gram_min_rows"] and cdiv(rows, R) * N < 2 * sms and
           cdiv(rows, R // 2) * n_out * 4 <= (K["gram_slab_mb"] << 20)):
        R //= 2
    chunks = cdiv(rows, R)
    I2 = (I + 1) & ~1
    return GramPlan(rows, R, chunks, rows - (chunks - 1) * R, chunks == 1, R * (I2 + J) * 2)


# X = Y: the engine's forward F = phi^T g (ldx = ldy = C, I = c, J = C, alpha 1);
# X != Y: its backward dF = (W/H) theta^T df over every pixel.  ldx / ldy > I / J put POISON in
# the padding.
GramCase = namedtuple("GramCase", "name N H W sub I J ldx ldy same")
GRAM_CASES = [
    GramCase("odd_i_bwd", 16, 28, 28, 1, 47, 96, 96, 96, False),
    GramCase("sub2_odd_h_ne_w", 4, 13, 11, 2, 10, 40, 40, 40, True),
    GramCase("padded_bwd", 8, 14, 10, 1, 9, 24, 40, 32, False),
    GramCase("padded_sub2", 6, 9, 15, 2, 7, 16, 24, 24, True),
    GramCase("direct", 300, 7, 7, 1, 16, 32, 32, 32, True),
    GramCase("r24_last_row", 88, 7, 7, 1, 9, 16, 16, 16, True),
    GramCase("r12_last_row", 4, 7, 7, 1, 6, 8, 8, 8, False),
    GramCase("slab_cap_r24", 64, 7, 7, 1, 40, 328, 328, 328, False),
    GramCase("r64", 64, 28, 28, 1, 40, 80, 80, 80, True),
    GramCase("r32", 16, 28, 28, 1, 40, 80, 80, 80, False),
    GramCase("r16", 8, 28, 28, 1, 24, 48, 48, 48, True),
    GramCase("n65535_1x1", 65535, 1, 1, 1, 3, 4, 4, 4, False),
    GramCase("autonl_14x14_sub2", 32, 14, 14, 2, 48, 96, 96, 96, True),
]


def gram_alpha(c):
    return 1.0 if c.same else float(c.W) / float(c.H)


# ---- non-local row x matrix ----------------------------------------------------------------------
RowmatPlan = namedtuple("RowmatPlan", "rows R chunks last odd_last smem")


def rowmat_plan(N, H, W, sub, Kd, O, sms=H100_SMS):
    """nl_rowmat_launch: rows per CTA (32, 16 or 8) and whether the last chunk has an odd row
    count (its second row of the last pair is zero padding, never stored)."""
    rows = sub_size(H, sub) * sub_size(W, sub)
    R = K["rowmat_rows"]
    while R > K["rowmat_min_rows"] and cdiv(rows, R) * N < 2 * sms:
        R //= 2
    chunks = cdiv(rows, R)
    last = rows - (chunks - 1) * R
    return RowmatPlan(rows, R, chunks, last, last % 2 == 1, Kd * O * 4 + R * ((Kd + 1) & ~1) * 2)


# The four argument patterns of _NlTail.rowmat in engine.py:
#   apply : f = (W/H) theta F              Mat = F     (sk = O, so = 1), sub 1
#   theta : dl = dy + [(W/H) df F^T | dy]  Mat = F^T   (sk = 1, so = K), base, O_copy = C > O
#   phi   : dl[sub rows] += g dF^T         Mat = dF^T  (sk = 1, so = K), accumulate
#   g     : dl[sub rows] += phi dF         Mat = dF    (sk = O, so = 1), accumulate
# gap: extra floats between samples of Mat (mat_stride = K*O + gap, POISON there); xpad / opad:
# pitch padding of X (POISON) and of out (SENTINEL)
RowmatCase = namedtuple("RowmatCase", "name mode N H W sub K O gap xpad opad")
ROWMAT_CASES = [
    RowmatCase("apply_odd_k", "apply", 8, 13, 11, 1, 9, 40, 6, 7, 8),
    RowmatCase("apply_sub2", "apply", 4, 13, 13, 2, 10, 24, 0, 0, 0),
    RowmatCase("theta_s1", "theta", 8, 13, 11, 1, 40, 10, 4, 8, 8),
    RowmatCase("theta_s2", "theta", 3, 9, 7, 2, 24, 8, 0, 0, 8),
    RowmatCase("phi_s1", "phi", 8, 13, 11, 1, 40, 10, 2, 0, 0),
    RowmatCase("phi_s2", "phi", 5, 13, 11, 2, 40, 10, 0, 8, 8),
    RowmatCase("g_s2_odd_k", "g", 6, 15, 9, 2, 9, 40, 3, 7, 0),
    RowmatCase("g_s1", "g", 8, 13, 11, 1, 10, 40, 0, 0, 8),
    RowmatCase("r32", "apply", 16, 28, 28, 1, 40, 80, 0, 0, 0),
    RowmatCase("r16_odd_last", "phi", 8, 27, 27, 1, 80, 40, 0, 0, 0),
    RowmatCase("r8_odd_last", "g", 2, 13, 13, 1, 11, 24, 0, 0, 0),
    RowmatCase("smem_limit", "apply", 4, 56, 56, 1, 80, 688, 0, 0, 0),
    RowmatCase("autonl_dg_14x14", "g", 32, 14, 14, 2, 48, 96, 0, 0, 0),
    RowmatCase("autonl_theta_7x7", "theta", 64, 7, 7, 1, 160, 80, 0, 0, 0),
]


def rowmat_strides(c):
    """(sk, so, mat_stride) of a case."""
    if c.mode in ("theta", "phi"):
        return 1, c.K, c.K * c.O + c.gap
    return c.O, 1, c.K * c.O + c.gap


def rowmat_o_copy(c):
    """Width of the output row (base pass-through up to it in the theta mode)."""
    return c.K if c.mode == "theta" else c.O


def rowmat_smem_ok(Kd, O, R):
    return Kd * O * 4 + R * ((Kd + 1) & ~1) * 2 <= K["rowmat_smem_kb"] * 1024


# ---- InstanceNorm --------------------------------------------------------------------------------
Lane = namedtuple("Lane", "CG PX idle")


def lanes(C):
    """lane_of per 64-channel chunk: channel groups CG, pixel lanes PX, idle threads."""
    out = []
    T, Ch = K["kThreads"], K["kChunk"]
    for chunk in range(cdiv(C, Ch)):
        CG = min(C // 8 - chunk * (Ch // 8), Ch // 8)
        PX = T // CG
        out.append(Lane(CG, PX, T - CG * PX))
    return out


def lane_pixels(HW, PX, px):
    return cdiv(HW - px, PX) if px < HW else 0


def has_tail(HW, PX):
    """Some pixel lane has pixels left after the kUnroll * PX loop."""
    return any(lane_pixels(HW, PX, px) % K["kUnroll"] for px in range(PX))


def lane_chain(HW, PX):
    """Longest per-lane fp32 chain (pixels of one lane)."""
    return cdiv(HW, PX)


# ldh > C: POISON in h's padding, SENTINEL in y's / dh's; off: a large per-channel offset
# (|mean| >> std); res / res2: residual inputs; affine False: gamma / beta NULL; mom: momentum
# (0: no running statistics, no counter); grads: which of dgamma / dbeta the backward takes
InCase = namedtuple("InCase", "name N HW C ldpad off affine res res2 mom grads")
IN_CASES = [
    InCase("c8_hw2", 3, 2, 8, 0, 0.0, True, True, False, 0.1, "both"),
    InCase("c24_hw3", 65, 3, 24, 8, 0.0, True, False, True, 0.1, "dgamma"),
    InCase("c56_hw49", 3, 49, 56, 0, 100.0, False, True, True, 0.1, "dbeta"),
    InCase("c64_hw196", 1, 196, 64, 16, 0.0, True, False, False, 0.0, "none"),
    InCase("c72_hw784", 3, 784, 72, 8, 30.0, True, True, True, 0.1, "both"),
    InCase("c120_hw49", 65, 49, 120, 0, 0.0, True, True, False, 0.0, "both"),
    InCase("c320_hw196", 3, 196, 320, 8, 0.0, True, True, True, 0.25, "both"),
    InCase("c24_hw784", 1, 784, 24, 0, 500.0, True, False, True, 0.1, "both"),
    InCase("c56_hw2", 65, 2, 56, 8, 0.0, False, False, False, 0.1, "none"),
    InCase("c120_hw3", 1, 3, 120, 0, 0.0, True, True, True, 0.1, "dgamma"),
    InCase("c8_hw196", 65, 196, 8, 8, 0.0, True, False, False, 0.1, "both"),
    InCase("autonl_l_14x14", 32, 196, 96, 0, 0.0, True, True, True, 0.1, "both"),
]
