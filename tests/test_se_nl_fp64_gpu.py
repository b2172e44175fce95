"""GPU: the Squeeze-and-Excitation fully connected layers (yamb_se_fc_fwd / _bwd), the non-local
products (yamb_nl_gram_fwd, yamb_nl_rowmat_fwd) and the non-local InstanceNorm
(yamb_instance_norm_fwd / _bwd), called through the C ABI for every case of tests/se_nl_cases.py
and compared with a float64 reference on the device, element by element.  The bounds and the
staging convention are in tests/se_nl_ref64.py.

SE: rows 0.. of `pooled` are zero, so u = b_r exactly there; b_r starts with 0, -0, 6, -3, 3,
-100, 100, which puts act / act' at their edges and __expf at overflow.  Parameter gradients
accumulate onto non-zero values.  InstanceNorm: channel 0 is constant within each sample
(var = 0), channel 1 carries a large offset.  Inputs carry POISON in their pitch padding and in
the row after the last; outputs SENTINEL in theirs, in guard values after fp32 outputs and, for the
sub-sampled row x matrix product, on every row outside the row set: a kernel that writes there
fails.  Every entry point: two calls give the same bits, and the InstanceNorm arrival counter is
back to 0 after every call.

The sequence check runs a non-local block's six products through _NlTail.gram / _NlTail.rowmat
in the engine's order (sub 2, an odd map with H != W) and checks the final dl element by element,
with its three bf16 rounding points carried as intervals.

On failure the message names the element and where the launch plan put it.  With -s, each
entry point's largest err/bound and the share of bf16 outputs whose interval spans more than two
bf16 values are printed at the end."""
import ctypes as C

import pytest
import torch

import se_nl_cases as sc
import se_nl_ref64 as sr
from ref64 import (DEV, POISON, SENTINEL, _check_guard, _equal, _fail, _guarded, _nat, _same)

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
REPORT = {}


def _note(entry, ratio=None, share=None):
    r = REPORT.setdefault(entry, {"ratio": 0.0, "share": []})
    if ratio is not None:
        r["ratio"] = max(r["ratio"], ratio)
    if share is not None:
        r["share"].append(share)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run(fn, args):
    _nat().check(fn(C.byref(args), _nat().stream_handle()))
    torch.cuda.synchronize()


def _padded(M, width, ld, fill, gen, scale=1.0, dtype=BF):
    """[M + 1, ld]: random values in [:M, :width], `fill` elsewhere."""
    t = torch.full((M + 1, ld), fill, device=DEV, dtype=dtype)
    t[:M, :width] = (torch.randn(M, width, device=DEV, generator=gen) * scale).to(dtype)
    return t


# ---- Squeeze-and-Excitation ----------------------------------------------------------------------
def _se_locs(plan):
    sp = plan.split

    def split(n, j):
        return "(sample %d, column %d: tile (%d, %d) of %d, K in %d slabs of %d; finish CTA (%d, %d))" \
            % (n, j, n // 64, j // 64, sp.tiles, sp.nslab, sp.k_per_slab, j // 32, n // 8)

    def tile(m, j):
        return "(tile (%d, %d), K in one slab)" % (m // 64, j // 64)

    def col_dt(c):
        return "(channel %d: dt CTA column %d, %d slabs of 32 samples)" % (c, c // 256, plan.dt_slabs)

    def col_du(j):
        return "(column %d: finish CTA column %d, %d slabs of 8 samples)" % (j, j // 32,
                                                                           plan.finish_slabs)
    return split, tile, col_dt, col_du


@pytest.mark.parametrize("c", sc.SE_CASES, ids=lambda c: c.name)
def test_se_fc(built_lib, c):
    nat = _nat()
    N, Cc, R, act = c.N, c.C, c.R, c.act
    plan = sc.se_plan(N, Cc, R, _sms())
    split, tile, col_dt, col_du = _se_locs(plan)
    g = torch.Generator(device=DEV).manual_seed(N * 7 + Cc * 3 + R + act)
    rnd = lambda *s, k=1.0: torch.randn(*s, device=DEV, generator=g) * k   # noqa: E731
    pooled = rnd(N, Cc)
    pooled[:min(N, 3)] = 0.0
    w_r, b_r = rnd(R, Cc, k=2 * Cc ** -0.5), rnd(R, k=0.5)
    ne = min(R, len(sc.SE_ACT_EDGES))
    b_r[:ne] = torch.tensor(sc.SE_ACT_EDGES[:ne], device=DEV)
    w_e, b_e = rnd(Cc, R, k=2 * R ** -0.5), rnd(Cc, k=0.5)
    what = "se_fc %s" % c.name

    def fwd():
        o = {k: _guarded(n, SENTINEL) for k, n in (("u", N * R), ("v", N * R), ("gate", N * Cc))}
        f = nat.SeFc()
        f.N, f.C, f.R, f.act = N, Cc, R, act
        f.pooled, f.w_r, f.b_r, f.w_e, f.b_e = (t.data_ptr() for t in (pooled, w_r, b_r, w_e, b_e))
        f.u, f.v, f.gate = o["u"].data_ptr(), o["v"].data_ptr(), o["gate"].data_ptr()
        _run(built_lib.yamb_se_fc_fwd, f)
        for k, n in (("u", N * R), ("v", N * R), ("gate", N * Cc)):
            _check_guard(o[k], n, what + " " + k)
        return o

    o = fwd()
    for k, t in fwd().items():
        _same(o[k], t, what + " " + k)
    u, v, gate = o["u"][:N * R].view(N, R), o["v"][:N * R].view(N, R), o["gate"][:N * Cc].view(N, Cc)
    _note("se_fc_fwd", sr.se_u_check(pooled, w_r, b_r, u, plan, what + " u", split))
    _equal(u[:min(N, 3)], b_r.expand(min(N, 3), R), what + " u on the pooled = 0 rows", split)
    _note("se_fc_fwd", sr.se_v_check(u, v, act, what + " v", split))
    _note("se_fc_fwd", sr.se_gate_check(v, w_e, b_e, gate, what + " gate", tile))

    dgate = rnd(N, Cc)
    inv_hw = 1.0 / 49
    g0 = {"wr": rnd(R, Cc), "br": rnd(R), "we": rnd(Cc, R), "be": rnd(Cc)}

    def bwd():
        o = {k: _guarded(n, SENTINEL) for k, n in (("dpool", N * Cc), ("dt", N * Cc), ("du", N * R))}
        for k, t in g0.items():
            o[k] = _guarded(t.numel(), SENTINEL)
            o[k][:t.numel()] = t.view(-1)
        b = nat.SeFcBwd()
        b.N, b.C, b.R, b.act, b.inv_hw = N, Cc, R, act, inv_hw
        b.dgate, b.gate, b.u, b.v = dgate.data_ptr(), gate.data_ptr(), u.data_ptr(), v.data_ptr()
        b.pooled, b.w_r, b.w_e = pooled.data_ptr(), w_r.data_ptr(), w_e.data_ptr()
        b.dpool, b.dt, b.du = o["dpool"].data_ptr(), o["dt"].data_ptr(), o["du"].data_ptr()
        b.g_wr, b.g_br, b.g_we, b.g_be = (o[k].data_ptr() for k in ("wr", "br", "we", "be"))
        _run(built_lib.yamb_se_fc_bwd, b)
        for k, n in (("dpool", N * Cc), ("dt", N * Cc), ("du", N * R)):
            _check_guard(o[k], n, what + " " + k)
        for k, t in g0.items():
            _check_guard(o[k], t.numel(), what + " g_" + k)
        return o

    o = bwd()
    for k, t in bwd().items():
        _same(o[k], t, what + " bwd " + k)
    dt, du = o["dt"][:N * Cc].view(N, Cc), o["du"][:N * R].view(N, R)
    sr.se_dt_check(dgate, gate, dt, what + " dt", tile)
    r = [sr.colsum_check(o["be"][:Cc], g0["be"], dt, sc.K["se_dt_rows"], plan.dt_slabs,
                         what + " g_be", col_dt),
         sr.se_du_check(dt, w_e, u, act, du, plan, what + " du", split),
         sr.colsum_check(o["br"][:R], g0["br"], du, sc.K["se_finish_rows"], plan.finish_slabs,
                         what + " g_br", col_du),
         sr.se_dpool_check(du, w_r, inv_hw, o["dpool"][:N * Cc].view(N, Cc), what + " dpool", tile),
         sr.gemm_acc_check(o["we"][:Cc * R].view(Cc, R), g0["we"], dt, v, what + " g_we", tile),
         sr.gemm_acc_check(o["wr"][:R * Cc].view(R, Cc), g0["wr"], du, pooled, what + " g_wr", tile)]
    _note("se_fc_bwd", max(r))
    print("%s: plan %s; fwd/bwd err/bound %.3g" % (what, tuple(plan.split), max(r)))


# ---- non-local gram ------------------------------------------------------------------------------
@pytest.mark.parametrize("c", sc.GRAM_CASES, ids=lambda c: c.name)
def test_nl_gram(built_lib, c):
    nat = _nat()
    plan = sc.gram_plan(c.N, c.H, c.W, c.sub, c.I, c.J, _sms())
    M = c.N * c.H * c.W
    g = torch.Generator(device=DEV).manual_seed(c.N + c.H * 31 + c.I * 7 + c.J)
    if c.same:
        assert c.ldx == c.ldy and c.I <= c.J
        X = Y = _padded(M, c.J, c.ldy, POISON, g)
    else:
        X = _padded(M, c.I, c.ldx, POISON, g)
        Y = _padded(M, c.J, c.ldy, POISON, g)
    alpha = sc.gram_alpha(c)
    n = c.N * c.I * c.J

    def run():
        G = _guarded(n, SENTINEL)
        a = nat.NlGram()
        a.N, a.H, a.W, a.sub = c.N, c.H, c.W, c.sub
        a.X, a.ldx, a.I = X.data_ptr(), c.ldx, c.I
        a.Y, a.ldy, a.J = Y.data_ptr(), c.ldy, c.J
        a.alpha, a.G = alpha, G.data_ptr()
        _run(built_lib.yamb_nl_gram_fwd, a)
        _check_guard(G, n, "nl_gram G")
        return G

    G = run()
    _same(G, run(), "nl_gram G")

    def loc(s, i, j):
        return "(sample %d: CTAs (0..%d, %d), %d row chunks of %d rows, the last %d; %s)" % (
            s, plan.chunks - 1, s, plan.chunks, plan.R, plan.last,
            "direct store" if plan.direct else "chunk slabs added by det_reduce")
    r = sr.gram_check(G[:n], X, Y, c.N, c.H, c.W, c.sub, c.I, c.J, alpha, plan,
                      "nl_gram %s" % c.name, loc)
    _note("nl_gram_fwd", r)
    print("nl_gram %s: %s err/bound %.3g" % (c.name, tuple(plan), r))


# ---- non-local row x matrix ----------------------------------------------------------------------
def _rowmat_mat(N, Kd, O, sk, so, stride, g):
    """Mat [N * stride + 8] fp32, POISON where no (k, o) of the strides lands; and its [N, K, O]."""
    vals = torch.randn(N, Kd, O, device=DEV, generator=g) * Kd ** -0.5
    flat = torch.full((N * stride + 8,), POISON, device=DEV)
    idx = (torch.arange(Kd, device=DEV)[:, None] * sk + torch.arange(O, device=DEV)[None, :] * so)
    off = torch.arange(N, device=DEV)[:, None, None] * stride + idx
    flat[off.reshape(-1)] = vals.reshape(-1)
    return flat, vals.double()


def _rowmat_loc(plan):
    def loc(s, r, o):
        return "(sample %d, row %d, column %d: chunk %d of %d (%d rows, the last %d), CTA (%d, %d))" \
            % (s, r, o, r // plan.R, plan.chunks, plan.R, plan.last, r // plan.R, s)
    return loc


def _rowmat_args(N, H, W, sub, X, ldx, Kd, Mat, stride, sk, so, O, alpha, out, ldo, base=None,
                 ldb=0, o_copy=0, accumulate=0):
    r = _nat().NlRowmat()
    r.N, r.H, r.W, r.sub = N, H, W, sub
    r.X, r.ldx, r.K = X.data_ptr(), ldx, Kd
    r.Mat, r.mat_stride, r.sk, r.so, r.O = Mat.data_ptr(), stride, sk, so, O
    r.alpha = alpha
    if base is not None:
        r.base, r.ldb, r.O_copy = base.data_ptr(), ldb, o_copy
    r.accumulate = accumulate
    r.out, r.ldo = out.data_ptr(), ldo
    return r


@pytest.mark.parametrize("c", sc.ROWMAT_CASES, ids=lambda c: c.name)
def test_nl_rowmat(built_lib, c):
    N, H, W, sub, Kd, O = c.N, c.H, c.W, c.sub, c.K, c.O
    plan = sc.rowmat_plan(N, H, W, sub, Kd, O, _sms())
    M = N * H * W
    g = torch.Generator(device=DEV).manual_seed(N * 3 + H * 17 + Kd * 5 + O)
    sk, so, stride = sc.rowmat_strides(c)
    ocp = sc.rowmat_o_copy(c)
    ldx, ldo = Kd + c.xpad, ocp + c.opad
    X = _padded(M, Kd, ldx, POISON, g)
    Mat, M3 = _rowmat_mat(N, Kd, O, sk, so, stride, g)
    out0 = torch.full((M + 1, ldo), SENTINEL, device=DEV, dtype=BF)
    rows = sr.row_mask(N, H, W, sub, DEV).nonzero().view(-1)
    accumulate = c.mode in ("phi", "g")
    base = None
    if accumulate:
        out0[rows, :O] = torch.randn(rows.numel(), O, device=DEV, generator=g).to(BF)
    if c.mode == "theta":
        base = _padded(M, ocp, ldo, POISON, g)
    alpha = float(W) / float(H) if c.mode in ("apply", "theta") else 1.0

    def run():
        out = out0.clone()
        _run(built_lib.yamb_nl_rowmat_fwd,
             _rowmat_args(N, H, W, sub, X, ldx, Kd, Mat, stride, sk, so, O, alpha, out, ldo, base,
                          ldo, ocp, int(accumulate)))
        return out

    out = run()
    _same(out, run(), "nl_rowmat out")
    what = "nl_rowmat %s" % c.name
    y64, delta = sr.rowmat_check(out, out0, X, M3, N, H, W, sub, Kd, O, alpha, base, accumulate,
                                 ocp, what, _rowmat_loc(plan))
    share = sr.span_share(y64, delta)
    rows_out = out[rows, :O].view_as(y64)
    _note("nl_rowmat_fwd", sr.bf16_ratio(rows_out, y64, delta), share)
    print("%s: %s; bf16 intervals wider than two values: %.2f %%" % (what, tuple(plan), 100 * share))


# ---- InstanceNorm --------------------------------------------------------------------------------
def _in_loc(Cc, HW):
    lanes = sc.lanes(Cc)
    chunks = len(lanes)

    def loc(n, i, ch):
        ln = lanes[ch // sc.K["kChunk"]]
        px = i % ln.PX
        unrolled = (i // ln.PX) < sc.lane_pixels(HW, ln.PX, px) // sc.K["kUnroll"] * sc.K["kUnroll"]
        return "(sample %d, pixel %d, channel %d: CTA %d, group %d of %d, pixel lane %d of %d, %s)" % (
            n, i, ch, n * chunks + ch // sc.K["kChunk"], (ch % sc.K["kChunk"]) // 8, ln.CG, px, ln.PX,
            "unrolled loop" if unrolled else "tail")
    return loc


def _in_stat_loc(Cc):
    chunks = len(sc.lanes(Cc))
    return lambda n, ch: "(sample %d, channel %d: CTA %d)" % (n, ch, n * chunks + ch // sc.K["kChunk"])


@pytest.mark.parametrize("c", sc.IN_CASES, ids=lambda c: c.name)
def test_instance_norm(built_lib, c):
    nat = _nat()
    N, HW, Cc = c.N, c.HW, c.C
    M, ld = N * HW, Cc + c.ldpad
    lanes = sc.lanes(Cc)
    g = torch.Generator(device=DEV).manual_seed(N * 11 + HW * 3 + Cc)
    hv = torch.randn(N, HW, Cc, device=DEV, generator=g) * 2 + \
        c.off * (torch.rand(Cc, device=DEV, generator=g) + 0.5)
    hv[:, :, 0] = torch.randn(N, 1, device=DEV, generator=g) * 3          # var = 0
    hv[:, :, 1] += 1000.0                                                    # |mean| >> std
    h = torch.full((M + 1, ld), POISON, device=DEV, dtype=BF)
    h[:M, :Cc] = hv.reshape(M, Cc).to(BF)
    res = _padded(M, Cc, ld, POISON, g) if c.res else None
    res2 = _padded(M, Cc, ld, POISON, g) if c.res2 else None
    gamma = (torch.rand(Cc, device=DEV, generator=g) + 0.5) if c.affine else None
    beta = torch.randn(Cc, device=DEV, generator=g) if c.affine else None
    rm0 = torch.randn(Cc, device=DEV, generator=g)
    rv0 = torch.rand(Cc, device=DEV, generator=g) + 0.5
    eps = 1e-3
    counter = torch.zeros(1, device=DEV, dtype=torch.int32)
    what = "instance_norm %s" % c.name
    loc, sloc = _in_loc(Cc, HW), _in_stat_loc(Cc)

    def fwd():
        o = {"y": torch.full((M + 1, ld), SENTINEL, device=DEV, dtype=BF),
             "mean": _guarded(N * Cc, SENTINEL), "invstd": _guarded(N * Cc, SENTINEL),
             "rm": _guarded(Cc, SENTINEL), "rv": _guarded(Cc, SENTINEL)}
        o["rm"][:Cc], o["rv"][:Cc] = rm0, rv0
        s = nat.InFwd()
        s.N, s.HW, s.C, s.ldh = N, HW, Cc, ld
        s.h, s.gamma, s.beta = h.data_ptr(), nat.ptr(gamma), nat.ptr(beta)
        s.eps, s.momentum = eps, c.mom
        s.running_mean, s.running_var = o["rm"].data_ptr(), o["rv"].data_ptr()
        s.mean, s.invstd = o["mean"].data_ptr(), o["invstd"].data_ptr()
        s.residual, s.ldr = nat.ptr(res), ld
        s.residual2, s.ldr2 = nat.ptr(res2), ld
        s.y, s.ldy = o["y"].data_ptr(), ld
        s.counter = counter.data_ptr() if c.mom != 0 else None
        _run(built_lib.yamb_instance_norm_fwd, s)
        assert int(counter.item()) == 0, what + ": arrival counter not back to 0"
        for k, n in (("mean", N * Cc), ("invstd", N * Cc), ("rm", Cc), ("rv", Cc)):
            _check_guard(o[k], n, what + " " + k)
        return o

    o = fwd()
    for k, t in fwd().items():
        _same(o[k], t, what + " " + k)
    y = o["y"]
    assert bool((y[:M, Cc:] == SENTINEL).all()) and bool((y[M] == SENTINEL).all()), \
        what + ": y written outside [M, C)"
    mean, invstd = o["mean"][:N * Cc].view(N, Cc), o["invstd"][:N * Cc].view(N, Cc)
    _, _, e_mean, e_var, rs = sr.in_stats_check(h, N, HW, Cc, eps, mean, invstd, lanes, what, sloc)
    y64, delta = sr.in_y_check(h, N, HW, Cc, gamma, beta, mean, invstd, res, res2, y, what, loc)
    _note("instance_norm_fwd", rs, sr.span_share(y64, delta))
    _note("instance_norm_fwd", sr.bf16_ratio(y[:M, :Cc].view(N, HW, Cc), y64, delta))
    if c.mom == 0:
        _same(o["rm"][:Cc], rm0, what + " running_mean without momentum")
        _same(o["rv"][:Cc], rv0, what + " running_var without momentum")
    else:
        _note("instance_norm_fwd", sr.in_running_check(h, N, HW, Cc, eps, c.mom, c.affine, rm0, rv0,
                                                       o["rm"][:Cc], o["rv"][:Cc], e_mean, e_var,
                                                       what))

    dy = _padded(M, Cc, ld, POISON, g)
    dg0, db0 = torch.randn(Cc, device=DEV, generator=g), torch.randn(Cc, device=DEV, generator=g)

    def bwd(grads):
        o = {"dh": torch.full((M + 1, ld), SENTINEL, device=DEV, dtype=BF),
             "dg": _guarded(Cc, SENTINEL), "db": _guarded(Cc, SENTINEL)}
        o["dg"][:Cc], o["db"][:Cc] = dg0, db0
        s = nat.InBwd()
        s.N, s.HW, s.C = N, HW, Cc
        s.ldh = s.lddy = s.lddh = ld
        s.dy, s.h, s.gamma = dy.data_ptr(), h.data_ptr(), nat.ptr(gamma)
        s.mean, s.invstd = mean.data_ptr(), invstd.data_ptr()
        s.dgamma = o["dg"].data_ptr() if grads in ("both", "dgamma") else None
        s.dbeta = o["db"].data_ptr() if grads in ("both", "dbeta") else None
        s.dh = o["dh"].data_ptr()
        s.counter = counter.data_ptr() if grads != "none" else None
        _run(built_lib.yamb_instance_norm_bwd, s)
        assert int(counter.item()) == 0, what + ": arrival counter not back to 0"
        _check_guard(o["dg"], Cc, what + " dgamma")
        _check_guard(o["db"], Cc, what + " dbeta")
        return o

    o = bwd(c.grads)
    for k, t in bwd(c.grads).items():
        _same(o[k], t, what + " bwd " + k)
    if c.grads != "none":
        _same(o["dh"], bwd("none")["dh"], what + " dh with and without dgamma / dbeta")
    dh = o["dh"]
    assert bool((dh[:M, Cc:] == SENTINEL).all()) and bool((dh[M] == SENTINEL).all()), \
        what + ": dh written outside [M, C)"
    S, Qr, e_S, e_Qr, dh64, dd = sr.in_bwd_check(dy, h, N, HW, Cc, gamma, mean, invstd, dh, lanes,
                                                 what, loc)
    _note("instance_norm_bwd", sr.bf16_ratio(dh[:M, :Cc].view(N, HW, Cc), dh64, dd),
          sr.span_share(dh64, dd))
    print("%s: bf16 intervals wider than two values: y %.2f %%, dh %.2f %%" % (
        what, 100 * sr.span_share(y64, delta), 100 * sr.span_share(dh64, dd)))
    if c.grads in ("both", "dgamma"):
        _note("instance_norm_bwd", sr.in_param_check(o["dg"][:Cc], dg0, Qr, e_Qr, what + " dgamma"))
    else:
        _same(o["dg"][:Cc], dg0, what + " dgamma not requested")
    if c.grads in ("both", "dbeta"):
        _note("instance_norm_bwd", sr.in_param_check(o["db"][:Cc], db0, S, e_S, what + " dbeta"))
    else:
        _same(o["db"][:Cc], db0, what + " dbeta not requested")


# ---- the non-local block's sequence through the engine's argument builders ------------------------
def _bf_round(t):
    return t.float().to(BF).double()


def _step(lo, hi, r, A, Kd):
    """The bf16 interval after out = bf16(out + r') with out in [lo, hi], |r' - r| within the
    K-fma chain, the add rounding to fp32 first."""
    d = 1.02 * (sr.gam(Kd) * A + sr.U * r.abs() + sr.U * (r.abs() + torch.maximum(lo.abs(),
                                                                                   hi.abs())))
    return _bf_round(lo + r - d), _bf_round(hi + r + d)


def test_nl_tail_sequence(built_lib):
    from yet_another_mobilenet_series_b200 import engine
    N, H, W, Cc, cr, sub = 3, 11, 9, 40, 10, 2
    M = N * H * W
    t = engine._NlTail.__new__(engine._NlTail)
    t.N, t.H, t.W, t.C, t.M, t.cr, t.sub = N, H, W, Cc, M, cr, sub
    t.scale = float(W) / float(H)
    g = torch.Generator(device=DEV).manual_seed(7)
    l, df, dym = (torch.randn(M, Cc, device=DEV, generator=g).to(BF) for _ in range(3))
    F, dF = _guarded(N * cr * Cc, SENTINEL), _guarded(N * cr * Cc, SENTINEL)
    f = torch.full((M + 1, Cc), SENTINEL, device=DEV, dtype=BF)
    dl = torch.full((M + 1, Cc), SENTINEL, device=DEV, dtype=BF)
    t.gram(l, cr, l, sub, 1.0, F, "nl_gram")
    t.rowmat(l, cr, F, Cc, 1, Cc, 1, t.scale, f, "nl_apply")
    t.gram(l, cr, df, 1, t.scale, dF, "nl_gram_bwd")
    t.rowmat(df, Cc, F, 1, Cc, cr, 1, t.scale, dl, "nl_dtheta", base=dym)
    t.rowmat(l, Cc, dF, 1, Cc, cr, t.sub, 1.0, dl, "nl_dphi", accumulate=1)
    t.rowmat(l, cr, dF, Cc, 1, Cc, t.sub, 1.0, dl, "nl_dg", accumulate=1)
    torch.cuda.synchronize()
    sms = _sms()
    _check_guard(F, N * cr * Cc, "sequence F")
    _check_guard(dF, N * cr * Cc, "sequence dF")
    sr.gram_check(F[:N * cr * Cc], l, l, N, H, W, sub, cr, Cc, 1.0,
                  sc.gram_plan(N, H, W, sub, cr, Cc, sms), "sequence F")
    sr.gram_check(dF[:N * cr * Cc], l, df, N, H, W, 1, cr, Cc, t.scale,
                  sc.gram_plan(N, H, W, 1, cr, Cc, sms), "sequence dF")
    F3 = F[:N * cr * Cc].double().view(N, cr, Cc)
    dF3 = dF[:N * cr * Cc].double().view(N, cr, Cc)
    f0 = torch.full_like(f, SENTINEL)
    sr.rowmat_check(f, f0, l, F3, N, H, W, 1, cr, Cc, t.scale, None, False, Cc, "sequence f")
    # dl = dy + [(W/H) df F^T | 0], then the row set += g dF^T on [:c], += phi dF
    r1, A1 = sr.rowmat_value(df, F3.transpose(1, 2), N, H, W, 1, Cc, t.scale)
    b1 = dym.double().view(N, H * W, Cc)[:, :, :cr]
    d1 = sr.rowmat_delta(r1, A1, b1, Cc)
    lo = dym.double().view(N, H, W, Cc).clone()
    hi = lo.clone()
    lo[..., :cr] = _bf_round(r1 + b1 - d1).view(N, H, W, cr)
    hi[..., :cr] = _bf_round(r1 + b1 + d1).view(N, H, W, cr)
    lo_s, hi_s = lo[:, ::sub, ::sub].reshape(N, -1, Cc), hi[:, ::sub, ::sub].reshape(N, -1, Cc)
    r2, A2 = sr.rowmat_value(l, dF3.transpose(1, 2), N, H, W, sub, Cc, 1.0)
    lo_s[..., :cr], hi_s[..., :cr] = _step(lo_s[..., :cr], hi_s[..., :cr], r2, A2, Cc)
    r3, A3 = sr.rowmat_value(l, dF3, N, H, W, sub, cr, 1.0)
    lo_s, hi_s = _step(lo_s, hi_s, r3, A3, cr)
    Hs, Ws = sc.sub_size(H, sub), sc.sub_size(W, sub)
    lo[:, ::sub, ::sub] = lo_s.view(N, Hs, Ws, Cc)
    hi[:, ::sub, ::sub] = hi_s.view(N, Hs, Ws, Cc)
    got = dl[:M].double().view(N, H, W, Cc)
    bad = (got < lo) | (got > hi) | ~torch.isfinite(got)
    if bool(bad.any()):
        i = tuple(bad.nonzero()[0].tolist())
        _fail("sequence dl", i, lambda n, y, x, ch: "(sample %d, pixel (%d, %d), channel %d; %s)" % (
            n, y, x, ch, "in the row set" if y % sub == 0 and x % sub == 0 else "outside the row set"),
            "got %r outside [%r, %r] (%d elements)" % (float(got[i]), float(lo[i]), float(hi[i]),
                                                       int(bad.sum())))
    assert bool((dl[M] == SENTINEL).all()), "sequence dl: wrote the row after M"
    key = lambda v: torch.where(v.float().to(BF).view(torch.int16).int() >= 0,      # noqa: E731
                                v.float().to(BF).view(torch.int16).int(),
                                -(v.float().to(BF).view(torch.int16).int() & 0x7fff))
    share = float(((key(hi) - key(lo) + 1) > 2).double().mean())
    _note("nl_tail_sequence_dl", None, share)
    print("nl tail sequence: dl intervals wider than two bf16 values: %.2f %%" % (100 * share))


# ---- refused calls write nothing -----------------------------------------------------------------
def test_refused_calls_write_nothing(built_lib):
    nat = _nat()
    lib = built_lib
    sink = torch.full((1 << 23,), SENTINEL, device=DEV)
    bsink = torch.full((1 << 22,), SENTINEL, device=DEV, dtype=BF)
    p, bp = sink.data_ptr(), bsink.data_ptr()
    calls = []
    for N, Cc, R in ((4, 4097, 8), (4, 64, 1025), (sc.SE_MAX_N + 1, 8, 2)):
        f = nat.SeFc()
        f.N, f.C, f.R, f.act = N, Cc, R, 1
        f.pooled = f.w_r = f.b_r = f.w_e = f.b_e = f.u = f.v = f.gate = p
        calls.append((lib.yamb_se_fc_fwd, f))
        b = nat.SeFcBwd()
        b.N, b.C, b.R, b.act, b.inv_hw = N, Cc, R, 1, 0.5
        for k in ("dgate", "gate", "u", "v", "pooled", "w_r", "w_e", "dpool", "dt", "du", "g_wr",
                  "g_br", "g_we", "g_be"):
            setattr(b, k, p)
        calls.append((lib.yamb_se_fc_bwd, b))
    for J, ldy in ((5, 6), (4, 5)):
        a = nat.NlGram()
        a.N, a.H, a.W, a.sub = 2, 7, 7, 1
        a.X, a.ldx, a.I, a.Y, a.ldy, a.J = bp, 8, 4, bp, ldy, J
        a.alpha, a.G = 1.0, p
        calls.append((lib.yamb_nl_gram_fwd, a))
    for Kd, O, with_base, acc in ((8, 5, False, 0), (8, 8, True, 1), (80, 704, False, 0)):
        r = _rowmat_args(2, 7, 7, 1, bsink, Kd, Kd, sink, Kd * O, O, 1, O, 1.0, bsink, O + 2,
                         bsink if with_base else None, O + 2, O + 2, acc)
        calls.append((lib.yamb_nl_rowmat_fwd, r))
    for N, HW, Cc in ((2, 1, 16), (2, 49, 12)):
        s = nat.InFwd()
        s.N, s.HW, s.C, s.ldh, s.ldr, s.ldr2, s.ldy = N, HW, Cc, 16, 16, 16, 16
        s.h = s.residual = s.residual2 = s.y = bp
        s.gamma = s.beta = s.running_mean = s.running_var = s.mean = s.invstd = p
        s.eps, s.momentum, s.counter = 1e-3, 0.1, p
        calls.append((lib.yamb_instance_norm_fwd, s))
        d = nat.InBwd()
        d.N, d.HW, d.C, d.ldh, d.lddy, d.lddh = N, HW, Cc, 16, 16, 16
        d.dy = d.h = d.dh = bp
        d.gamma = d.mean = d.invstd = d.dgamma = d.dbeta = d.counter = p
        calls.append((lib.yamb_instance_norm_bwd, d))
    for fn, args in calls:
        rc = fn(C.byref(args), nat.stream_handle())
        assert rc == nat.EINVAL, (fn.__name__, rc, lib.yamb_last_error())
    torch.cuda.synchronize()
    assert bool((sink == SENTINEL).all()), "a refused call wrote an fp32 buffer"
    assert bool((bsink == SENTINEL).all()), "a refused call wrote a bf16 buffer"


def test_report():
    """Largest err/bound per entry point and the share of bf16 outputs whose interval holds more
    than two bf16 values (shown with -s; nothing to assert)."""
    for k in sorted(REPORT):
        r = REPORT[k]
        s = ("bf16 wider than two values: up to %.2f %%" % (100 * max(r["share"]))
             if r["share"] else "")
        print("%-22s max err/bound %.3g  %s" % (k, r["ratio"], s))
