"""CPU: the launch-plan mirror of tests/se_nl_cases.py against the kernel sources, the reach of the
case tables of test_se_nl_fp64_gpu.py over every branch of those plans, and the element checkers
of tests/se_nl_ref64.py against planted faults.  A checker must pass the exact fp64 reference
rounded to the output type and fail on each planted fault: that is the evidence that its bounds
are tight enough to see the faults the GPU test exists for."""
import pytest
import torch

import se_nl_cases as sc
import se_nl_ref64 as sr
from ref64 import SENTINEL

BF = torch.bfloat16


# ---- constants -----------------------------------------------------------------------------------
def test_constants_match_the_sources():
    assert sc.parse_constants() == sc.K


def test_parser_sees_a_changed_constant(tmp_path):
    with open(sc.IN_SOURCE) as f:
        src = f.read()
    p = tmp_path / "instance_norm.cu"
    p.write_text(src.replace("constexpr int kUnroll = 4;", "constexpr int kUnroll = 2;"))
    assert sc.parse_constants(inorm=str(p))["kUnroll"] == 2
    with open(sc.NL_SOURCE) as f:
        src = f.read()
    p = tmp_path / "nonlocal.cu"
    p.write_text(src.replace("int R = 32;", "int R = 64;"))
    assert sc.parse_constants(nl=str(p))["rowmat_rows"] == 64


# ---- coverage ------------------------------------------------------------------------------------
def _se_needs():
    need = {
        "one K slab, C <= 64": lambda c, p: p.split.nslab == 1 and c.C <= 64,
        "one K slab, enough tiles": lambda c, p: p.split.nslab == 1 and c.C > 4 * sc.K["kSgK"],
        "several K slabs": lambda c, p: p.split.nslab > 1,
        "fewer K slabs than ksplit": lambda c, p: 1 < p.split.nslab < p.split.ksplit,
        "C not a multiple of 16": lambda c, p: c.C % sc.K["kSgK"] != 0,
        "R not a multiple of 16": lambda c, p: c.R % sc.K["kSgK"] != 0,
        "N, R not multiples of 64, several tiles in M and N": lambda c, p: c.N > 64 and c.C > 64 and
        c.R > 64 and c.N % 64 and c.R % 64,
        "N % 8 != 0 over several finish slabs": lambda c, p: c.N % 8 and p.finish_slabs > 1,
        "N % 32 != 0 over several dt slabs": lambda c, p: c.N % 32 and p.dt_slabs > 1,
        "C = 4096": lambda c, p: c.C == sc.K["se_max_c"],
        "N = 8 x 65535": lambda c, p: c.N == sc.SE_MAX_N,
        "AutoNL-L": lambda c, p: (c.C, c.R) in sc.AUTONL_L_SE,
    }
    for cr in sc.ATOMNAS_CP_SE:
        need["AtomNAS-C+ %s" % (cr,)] = lambda c, p, cr=cr: (c.C, c.R) == cr
    for a in range(5):
        need["act %d" % a] = lambda c, p, a=a: c.act == a
    for n in (1, 7, 8, 9, 31, 32, 33):
        need["N = %d" % n] = lambda c, p, n=n: c.N == n
    for r in (1, 2, 4, 10, 65, 1024):
        need["R = %d" % r] = lambda c, p, r=r: c.R == r
    return need


def _gram_needs(sms):
    need = {
        "odd I, even J": lambda c, p: c.I % 2 and c.J % 2 == 0,
        "sub 2, odd H and W": lambda c, p: c.sub == 2 and c.H % 2 and c.W % 2,
        "sub 2, H != W": lambda c, p: c.sub == 2 and c.H != c.W,
        "ldx > I": lambda c, p: c.ldx > c.I and not c.same,
        "ldy > J": lambda c, p: c.ldy > c.J,
        "one chunk (direct store)": lambda c, p: p.direct,
        "several chunks (det_reduce)": lambda c, p: not p.direct,
        "R not a power of two": lambda c, p: p.R & (p.R - 1),
        "last chunk of one row": lambda c, p: p.chunks > 1 and p.last == 1,
        "halving stopped by the slab cap": lambda c, p: p.R > sc.K["gram_min_rows"] and
        p.chunks * c.N < 2 * sms,
        "N = 65535 at 1x1": lambda c, p: c.N == 65535 and c.H == c.W == 1,
        "X = Y (forward)": lambda c, p: c.same,
        "X != Y (backward)": lambda c, p: not c.same,
    }
    for R in (64, 32, 16):
        need["R = %d" % R] = lambda c, p, R=R: p.R == R
    return need


def _rowmat_needs():
    need = {
        "odd K": lambda c, p: c.K % 2,
        "Mat gaps (mat_stride > K O)": lambda c, p: c.gap > 0,
        "X pitch > K": lambda c, p: c.xpad > 0,
        "out pitch > row width": lambda c, p: c.opad > 0,
        "odd last chunk": lambda c, p: p.odd_last,
        "O_copy > O": lambda c, p: c.mode == "theta" and sc.rowmat_o_copy(c) > c.O,
        "largest K O in shared memory": lambda c, p: p.smem <= sc.K["rowmat_smem_kb"] * 1024 and
        not sc.rowmat_smem_ok(c.K, c.O + 2, p.R),
        "transposed Mat (sk = 1)": lambda c, p: sc.rowmat_strides(c)[0] == 1,
    }
    for R in (32, 16, 8):
        need["R = %d" % R] = lambda c, p, R=R: p.R == R
    for mode in ("apply", "theta", "phi", "g"):
        for sub in (1, 2):
            need["%s, sub %d, odd map" % (mode, sub)] = lambda c, p, m=mode, s=sub: \
                c.mode == m and c.sub == s and (c.H % 2 or c.W % 2)
    return need


def _in_needs():
    need = {
        "HW < PX": lambda c: any(c.HW < ln.PX for ln in sc.lanes(c.C)),
        "tail after the unrolled loop": lambda c: any(sc.has_tail(c.HW, ln.PX)
                                                      for ln in sc.lanes(c.C)),
        "idle threads (PX does not divide 256)": lambda c: any(ln.idle for ln in sc.lanes(c.C)),
        "|mean| >> std": lambda c: c.off > 0,
        "gamma / beta NULL": lambda c: not c.affine,
        "residual": lambda c: c.res, "no residual": lambda c: not c.res,
        "residual2": lambda c: c.res2, "no residual2": lambda c: not c.res2,
        "pitch > C": lambda c: c.ldpad > 0,
        "momentum 0": lambda c: c.mom == 0, "momentum != 0": lambda c: c.mom != 0,
    }
    for C in (8, 24, 56, 64, 72, 120, 320):
        need["C = %d" % C] = lambda c, C=C: c.C == C
    for cg in (1, 3, 7, 8):
        need["CG = %d" % cg] = lambda c, cg=cg: any(ln.CG == cg for ln in sc.lanes(c.C))
    for hw in (2, 3, 49, 196, 784):
        need["HW = %d" % hw] = lambda c, hw=hw: c.HW == hw
    for n in (1, 3, 65):
        need["N = %d" % n] = lambda c, n=n: c.N == n
    for gr in ("both", "dgamma", "dbeta", "none"):
        need["grads %s" % gr] = lambda c, gr=gr: c.grads == gr
    return need


def _missing(sms):
    miss = []
    for k, pred in _se_needs().items():
        if not any(pred(c, sc.se_plan(c.N, c.C, c.R, sms)) for c in sc.SE_CASES):
            miss.append("se_fc: " + k)
    for k, pred in _gram_needs(sms).items():
        if not any(pred(c, sc.gram_plan(c.N, c.H, c.W, c.sub, c.I, c.J, sms)) for c in sc.GRAM_CASES):
            miss.append("nl_gram: " + k)
    for k, pred in _rowmat_needs().items():
        if not any(pred(c, sc.rowmat_plan(c.N, c.H, c.W, c.sub, c.K, c.O, sms))
                   for c in sc.ROWMAT_CASES):
            miss.append("nl_rowmat: " + k)
    for k, pred in _in_needs().items():
        if not any(pred(c) for c in sc.IN_CASES):
            miss.append("instance_norm: " + k)
    return miss


def test_tables_reach_every_branch_on_h100_sxm():
    assert _missing(sc.H100_SMS) == []


def test_tables_on_h100_pcie():
    """At 114 SMs only the split-K SE case with fewer slabs than ksplit moves (AtomNAS-C+'s 2310
    channels get 29 of 29 slabs); the smaller slab count of another case keeps the branch."""
    assert _missing(sc.H100_PCIE_SMS) == []
    moved = [c.name for c in sc.SE_CASES
             if sc.se_plan(c.N, c.C, c.R) != sc.se_plan(c.N, c.C, c.R, sc.H100_PCIE_SMS)]
    moved += [c.name for c in sc.GRAM_CASES
              if sc.gram_plan(c.N, c.H, c.W, c.sub, c.I, c.J) !=
              sc.gram_plan(c.N, c.H, c.W, c.sub, c.I, c.J, sc.H100_PCIE_SMS)]
    moved += [c.name for c in sc.ROWMAT_CASES
              if sc.rowmat_plan(c.N, c.H, c.W, c.sub, c.K, c.O) !=
              sc.rowmat_plan(c.N, c.H, c.W, c.sub, c.K, c.O, sc.H100_PCIE_SMS)]
    print("plans that differ at 114 SMs: %s" % moved)
    assert sorted(moved) == ["atomnas_cp_2310", "autonl_theta_7x7", "r1024"], moved


def test_cases_are_legal():
    for c in sc.SE_CASES:
        assert 0 < c.C <= sc.K["se_max_c"] and 0 < c.R <= sc.K["se_max_r"] and \
            0 < c.N <= sc.SE_MAX_N, c
    for c in sc.GRAM_CASES:
        assert c.J % 2 == 0 and c.ldy % 2 == 0 and c.I <= c.ldx and c.J <= c.ldy, c
        assert sc.gram_plan(c.N, c.H, c.W, c.sub, c.I, c.J).smem <= sc.K["gram_smem_kb"] * 1024
    for c in sc.ROWMAT_CASES:
        assert c.O % 2 == 0 and (sc.rowmat_o_copy(c) + c.opad) % 2 == 0, c
        for sms in (sc.H100_SMS, sc.H100_PCIE_SMS):
            p = sc.rowmat_plan(c.N, c.H, c.W, c.sub, c.K, c.O, sms)
            assert sc.rowmat_smem_ok(c.K, c.O, p.R), c
    for c in sc.IN_CASES:
        assert c.C % 8 == 0 and c.HW >= 2 and (c.C + c.ldpad) % 8 == 0, c
    for t in (sc.SE_CASES, sc.GRAM_CASES, sc.ROWMAT_CASES, sc.IN_CASES):
        assert len({c.name for c in t}) == len(t)


# ---- the checkers catch the faults they exist for -------------------------------------------------
def _g(seed):
    return torch.Generator().manual_seed(seed)


def _se_data(N, C, R, seed=0):
    g = _g(seed)
    return (torch.randn(N, C, generator=g), torch.randn(R, C, generator=g) * C ** -0.5,
            torch.randn(R, generator=g) * 0.5)


def test_se_product_dropped_k_chunk():
    N, C, R = 100, 200, 70
    pooled, w_r, b_r = _se_data(N, C, R)
    plan = sc.se_plan(N, C, R)
    assert plan.split.nslab > 1
    u64 = pooled.double() @ w_r.double().t() + b_r.double()
    sr.se_u_check(pooled, w_r, b_r, u64.float(), plan, "u")
    bad = u64.clone()
    bad[:64, :64] -= pooled[:64, 16:32].double() @ w_r[:64, 16:32].double().t()
    with pytest.raises(AssertionError):
        sr.se_u_check(pooled, w_r, b_r, bad.float(), plan, "u")
    # the backward's split-K product du (act none: du = W_e^T dt)
    dt = torch.randn(N, C, generator=_g(1))
    w_e = torch.randn(C, R, generator=_g(2)) * R ** -0.5
    u = torch.randn(N, R, generator=_g(3))
    du64 = dt.double() @ w_e.double()
    sr.se_du_check(dt, w_e, u, 0, du64.float(), plan, "du")
    bad = du64.clone()
    bad[64:, 64:] -= dt[64:, 48:64].double() @ w_e[48:64, 64:].double()
    with pytest.raises(AssertionError):
        sr.se_du_check(dt, w_e, u, 0, bad.float(), plan, "du")


def test_bias_gradient_dropped_sample_slab():
    N, C = 100, 40
    dt = torch.randn(N, C, generator=_g(4))
    g0 = torch.randn(C, generator=_g(5))
    slabs = sc.cdiv(N, sc.K["se_dt_rows"])
    good = (g0.double() + dt.double().sum(0)).float()
    sr.colsum_check(good, g0, dt, sc.K["se_dt_rows"], slabs, "g_be")
    bad = (g0.double() + dt.double().sum(0) - dt[32:64].double().sum(0)).float()
    with pytest.raises(AssertionError):
        sr.colsum_check(bad, g0, dt, sc.K["se_dt_rows"], slabs, "g_be")
    bad = (g0.double() + dt.double().sum(0) - dt[96:].double().sum(0)).float()   # the last 4
    with pytest.raises(AssertionError):
        sr.colsum_check(bad, g0, dt, sc.K["se_dt_rows"], slabs, "g_be")


@pytest.mark.parametrize("act,edge,wrong", [(1, 0.0, 1.0), (2, 6.0, 1.0), (2, 0.0, 1.0),
                                            (4, -3.0, -0.5), (4, 3.0, 1.5)])
def test_act_derivative_wrong_at_an_edge(act, edge, wrong):
    N, C, R = 9, 72, 10
    plan = sc.se_plan(N, C, R)
    dt = torch.randn(N, C, generator=_g(6))
    w_e = torch.randn(C, R, generator=_g(7)) * R ** -0.5
    u = torch.randn(N, R, generator=_g(8)) * 3
    u[0, 0] = edge
    a = dt.double() @ w_e.double()
    g = sr._dact64(u.double(), act)
    sr.se_du_check(dt, w_e, u, act, (a * g).float(), plan, "du")
    g[0, 0] = wrong
    with pytest.raises(AssertionError):
        sr.se_du_check(dt, w_e, u, act, (a * g).float(), plan, "du")


def _bf(shape, seed):
    return torch.randn(*shape, generator=_g(seed)).to(BF)


def test_gram_dropped_row_chunk():
    N, H, W, I, J = 2, 14, 14, 10, 16
    plan = sc.gram_plan(N, H, W, 1, I, J)
    assert plan.chunks > 2
    X, Y = _bf((N * H * W, I), 9), _bf((N * H * W, J), 10)
    xs, ys = sr.rows_of(X, N, H, W, 1, I), sr.rows_of(Y, N, H, W, 1, J)
    G = 0.75 * (xs.transpose(1, 2) @ ys)
    sr.gram_check(G.float(), X, Y, N, H, W, 1, I, J, 0.75, plan, "G")
    R = plan.R
    bad = G.clone()
    bad[1] -= 0.75 * (xs[1, R:2 * R].t() @ ys[1, R:2 * R])
    with pytest.raises(AssertionError):
        sr.gram_check(bad.float(), X, Y, N, H, W, 1, I, J, 0.75, plan, "G")


def _rowmat_out(N, H, W, sub, X, M3, Kd, O, alpha, accumulate, ldo, seed, shift=0):
    """out0 and a correct (or, with shift, X read one pixel off) out of the row x matrix product."""
    M = N * H * W
    out0 = torch.full((M + 1, ldo), SENTINEL, dtype=BF)
    idx = sr.row_mask(N, H, W, sub, "cpu").nonzero().view(-1)
    if accumulate:
        out0[idx, :O] = _bf((idx.numel(), O), seed)
    Xs = torch.roll(X, -shift, 0) if shift else X
    r, _ = sr.rowmat_value(Xs, M3, N, H, W, sub, Kd, alpha)
    b = out0[idx, :O].double().view_as(r) if accumulate else torch.zeros_like(r)
    out = out0.clone()
    out[idx, :O] = (r + b).reshape(-1, O).float().to(BF)
    return out0, out, idx


def test_rowmat_row_set_shifted_by_one_pixel():
    N, H, W, sub, Kd, O = 2, 9, 7, 2, 12, 8
    X = _bf((N * H * W + 1, Kd), 11)
    M3 = torch.randn(N, Kd, O, generator=_g(12), dtype=torch.float64)
    for acc in (False, True):
        out0, out, _ = _rowmat_out(N, H, W, sub, X, M3, Kd, O, 1.0, acc, O, 13)
        sr.rowmat_check(out, out0, X, M3, N, H, W, sub, Kd, O, 1.0, None, acc, O, "out")
        out0, bad, _ = _rowmat_out(N, H, W, sub, X, M3, Kd, O, 1.0, acc, O, 13, shift=1)
        with pytest.raises(AssertionError):
            sr.rowmat_check(bad, out0, X, M3, N, H, W, sub, Kd, O, 1.0, None, acc, O, "out")


def test_rowmat_strides_swapped():
    N, H, W, Kd = 2, 5, 7, 8
    X = _bf((N * H * W + 1, Kd), 14)
    M3 = torch.randn(N, Kd, Kd, generator=_g(15), dtype=torch.float64)
    out0, out, _ = _rowmat_out(N, H, W, 1, X, M3, Kd, Kd, 0.7, False, Kd, 0)
    sr.rowmat_check(out, out0, X, M3, N, H, W, 1, Kd, Kd, 0.7, None, False, Kd, "out")
    out0, bad, _ = _rowmat_out(N, H, W, 1, X, M3.transpose(1, 2), Kd, Kd, 0.7, False, Kd, 0)
    with pytest.raises(AssertionError):
        sr.rowmat_check(bad, out0, X, M3, N, H, W, 1, Kd, Kd, 0.7, None, False, Kd, "out")


def test_rowmat_accumulate_write_outside_the_row_set():
    N, H, W, sub, Kd, O = 2, 9, 9, 2, 6, 10
    X = _bf((N * H * W + 1, Kd), 16)
    M3 = torch.randn(N, Kd, O, generator=_g(17), dtype=torch.float64)
    out0, out, idx = _rowmat_out(N, H, W, sub, X, M3, Kd, O, 1.0, True, O + 2, 18)
    sr.rowmat_check(out, out0, X, M3, N, H, W, sub, Kd, O, 1.0, None, True, O, "out")
    bad = out.clone()
    bad[1, 3] = 0.5                       # pixel (0, 1) of sample 0: not in the ::2 row set
    assert 1 not in idx.tolist()
    with pytest.raises(AssertionError):
        sr.rowmat_check(bad, out0, X, M3, N, H, W, sub, Kd, O, 1.0, None, True, O, "out")
    bad = out.clone()
    bad[int(idx[5]), O] = 0.5             # a padding column of a row in the set
    with pytest.raises(AssertionError):
        sr.rowmat_check(bad, out0, X, M3, N, H, W, sub, Kd, O, 1.0, None, True, O, "out")


@pytest.mark.parametrize("C,HW", [(64, 196), (24, 49), (56, 784), (8, 3)])
def test_instance_norm_dropped_pixel_lane(C, HW):
    N = 2
    lanes = sc.lanes(C)
    h = (torch.randn(N * HW, C, generator=_g(19)) * 2 + 5).to(BF)
    hv = h.double().view(N, HW, C)
    mean = hv.mean(1)
    inv = (hv.var(1, unbiased=False) + float(torch.tensor(1e-3))).rsqrt()
    sr.in_stats_check(h, N, HW, C, 1e-3, mean.float(), inv.float(), lanes, "in")
    PX = lanes[0].PX
    keep = torch.ones(HW, dtype=torch.bool)
    keep[0::PX] = False                   # pixel lane 0 of channel chunk 0
    bad = mean.clone()
    bad[1, :8] = hv[1, keep, :8].sum(0) / HW
    with pytest.raises(AssertionError):
        sr.in_stats_check(h, N, HW, C, 1e-3, bad.float(), inv.float(), lanes, "in")
