"""GPU parity of the per-channel kernels of csrc/elementwise.cu (bn_apply, bn_stats, bn_reduce,
bn_bwd_apply, se_pool, se_bwd_reduce, se_bwd_apply) and of the BatchNorm bookkeeping they share
with the GEMM epilogues (csrc/bn_finalize.cuh), each entry point called directly and every output
compared with a float64 reference of the same operation, element by element.  The shapes and a
restatement of each launcher's grid rule are in tests/ew_cases.py.

Staged values.  z = fmaf(scale, h, shift) is reproduced by forming the sum in fp64 (the product of
an fp32 and a bf16 value is exact there) and rounding once to fp32; fmaf(ca, dz, fmaf(cb, h, cc))
the same way, one fp32 rounding per fmaf.

Exact cases.  With no activation, ReLU or ReLU6, bn_apply must give the value of a float32
emulation of its order of operations (fma -> clamp -> x gate -> + residual -> + residual2 -> RN
bf16), and bn_bwd_apply, se_bwd_apply, se_pool and se_bwd_reduce's staged operands those of theirs
(dz -> act' mask -> fmaf(ca, dz, fmaf(cb, h, cc)) -> RN bf16), equal as values.  Swish and h-swish
run on __expf / __fdividef: where the exact value lies within 2^-16 (relative) of a bf16 rounding
boundary the stored value may sit one bf16 ulp away; the checks take the bf16 values of the
exact result moved by that much (plus the fp32 roundings of the later steps) as the allowed range.

Long sums (sum h, sum h^2, sum dz, sum dz * xhat, pooled, dgate): with r the fp64 reference and
Q = sqrt(sum term^2),  |got - r| <= 2^-10 |r| + 2^-8 Q  (plus the staging ulps of Swish / h-swish
terms).  A missing tile of rows changes such a sum by a multiple of Q.  se_bwd_apply's statistics
are sums of the bf16 values it stores; they are also gated against the sums of the stored values
at the fp32 accumulation bound 2^-24 (rows per thread + 2) sum |term|, which the rounding of the
stored values would exceed.

Derived values (mean, invstd, scale, shift, running statistics, ca / cb / cc) carry the bound
propagated through the fp64 derivation, plus the fp32 rounding of the stored value.  The running
statistics are checked against torch.nn.BatchNorm2d itself (momentum, momentum=None cumulative
through num_batches_tracked, unbiased running_var); dgamma / dbeta are accumulated (+=) into
pre-filled buffers.

Every call also checks: the BatchNorm accumulator and the counter come back zero; an identical
second call from identical buffers gives identical bits; columns outside the channel slice and a
row after M keep a sentinel (and a poison row after M in the inputs does not leak into any
output); se_bwd_apply in place (dz == dy) gives the bits of the out-of-place call.  On failure the
message names the element (row, channel) and the CTA and pass of the grid walk that produced it."""
import ctypes as C

import pytest
import torch

import ew_cases as ec

pytestmark = pytest.mark.gpu

from ref64 import (  # noqa: F401
    BAND, DEV, POISON, SENTINEL, _Acc, _act64, _act_err, _between, _bf, _bn_bwd, _bwd_outputs,
    _check_bwd_finalize, _check_frame, _check_fwd_finalize, _check_guard, _clamp32, _dact64,
    _equal, _eval_mode_coeffs, _f32, _guarded, _long_bound, _nat, _same, _staged_band, _with_poison,
    _worst)


# ---- helpers -------------------------------------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _walk_loc(plan, batch):
    """Locator of the row-walk kernels (bn_stats / bn_reduce / bn_bwd_apply / se_bwd_apply)."""
    def loc(row, ch, *_):
        cg = ch // 8
        r0 = row % plan.rstep
        return "(row %d, channel %d: CTA %d, pixel lane %d, channel pass %d, iteration %d, row %d " \
               "of the batch)" % (row, ch, r0 // plan.px, r0 % plan.px, cg // 256,
                                   row // (batch * plan.rstep), (row // plan.rstep) % batch)
    return loc


def _chan_loc(plan):
    def loc(ch, *_):
        return "(channel %d: channel pass %d; %d CTAs, %d pixel lanes)" % (
            ch, (ch // 8) // 256, plan.grid, plan.px)
    return loc


# ================================================================================================
def test_tables_on_this_device(built_lib):
    """The case tables reach their paths with this GPU's SM count (they were laid out for 132)."""
    assert built_lib.yamb_max_ctas() == 4 * _sms()
    ec.check_tables(_sms())


# ---- bn_apply ----------------------------------------------------------------------------------
@pytest.mark.parametrize("c", ec.APPLY_CASES, ids=lambda c: "M%d-C%d-act%d-%s" % (c.M, c.C, c.act, c.why))
def test_bn_apply(built_lib, c):
    nat = _nat()
    plan = ec.apply_plan(c.M, c.C, _sms())
    g = torch.Generator(device=DEV).manual_seed(11)
    M, Cc, ld, c0 = c.M, c.C, c.ld, c.c0
    h = _with_poison(_bf((M, ld), 1.5, 0.3, g))
    scale = torch.rand(Cc, device=DEV, generator=g) + 0.5
    shift = torch.randn(Cc, device=DEV, generator=g) * 0.3
    res = _with_poison(_bf((M, ld), 1.0, 0.0, g)) if c.res else None
    res2 = _with_poison(_bf((M, ld), 1.0, 0.0, g)) if c.res2 else None
    nsamp = ec.cdiv(M, c.gate) if c.gate else 0
    gate = torch.rand(nsamp, Cc, device=DEV, generator=g) if c.gate else None
    sl = lambda t: t[:M, c0:c0 + Cc]

    def run():
        y = torch.full((M + 1, ld), SENTINEL, device=DEV, dtype=torch.bfloat16)
        a = nat.BnApply()
        a.M, a.C, a.ldh, a.ldr, a.ldy = M, Cc, ld, ld, ld
        a.h, a.scale, a.shift, a.act = h.data_ptr() + 2 * c0, scale.data_ptr(), shift.data_ptr(), c.act
        a.y = y.data_ptr() + 2 * c0
        if res is not None:
            a.residual = res.data_ptr() + 2 * c0
        if res2 is not None:
            a.residual2, a.ldr2 = res2.data_ptr() + 2 * c0, ld
        if gate is not None:
            a.gate, a.rows_per_sample = gate.data_ptr(), c.gate
        nat.check(built_lib.yamb_bn_apply_fwd(C.byref(a), nat.stream_handle()))
        torch.cuda.synchronize()
        return y

    y = run()
    _same(y, run(), "bn_apply y")
    _check_frame(y, M, c0, Cc, "bn_apply")

    def loc(row, ch):
        i = row * (Cc // 8) + ch // 8
        return "(CTA %d, pass %d of the grid-stride walk)" % ((i % plan.stride) // 256, i // plan.stride)

    h64 = sl(h).double()
    z32 = _f32(h64 * scale.double() + shift.double())
    g_rows = gate[torch.arange(M, device=DEV) // c.gate] if gate is not None else None
    if c.act in (0, 1, 2):
        v = _clamp32(z32, c.act)
        if g_rows is not None:
            v = v * g_rows
        if res is not None:
            v = v + sl(res).float()
        if res2 is not None:
            v = v + sl(res2).float()
        _equal(sl(y), v.to(torch.bfloat16), "bn_apply y", loc)
    else:
        a64 = _act64(z32, c.act)
        ag = a64 * (g_rows.double() if g_rows is not None else 1.0)
        y64, mag = ag.clone(), ag.abs()
        for r in (res, res2):
            if r is not None:
                y64 += sl(r).double()
                mag += sl(r).double().abs()
        _between(sl(y), y64, BAND * ag.abs() + 2.0 ** -22 * mag, "bn_apply y", loc)


# ---- bn_stats + forward finalize ---------------------------------------------------------------
@pytest.mark.parametrize("c", ec.STATS_CASES, ids=lambda c: "M%d-C%d-%s" % (c.M, c.C, c.why))
def test_bn_stats(built_lib, c):
    nat = _nat()
    plan = ec.stats_plan(c.M, c.C, _sms())
    g = torch.Generator(device=DEV).manual_seed(12)
    M, Cc, ld, c0 = c.M, c.C, c.ld, c.c0
    if c.data == "shifted":
        sig = torch.rand(Cc, device=DEV, generator=g) + 0.5
        sign = torch.randint(0, 2, (Cc,), device=DEV, generator=g) * 2 - 1
        mu = 20.0 * sig * (1 + 0.25 * torch.rand(Cc, device=DEV, generator=g)) * sign
        hs = torch.zeros(M, ld, device=DEV)
        hs[:, c0:c0 + Cc] = mu + sig * torch.randn(M, Cc, device=DEV, generator=g)
        h = _with_poison(hs.to(torch.bfloat16))
    else:
        h = _with_poison(_bf((M, ld), 1.5, 0.3, g))
    gamma = torch.rand(Cc, device=DEV, generator=g) + 0.5 if c.affine else None
    beta = torch.randn(Cc, device=DEV, generator=g) if c.affine else None
    rm0 = torch.randn(Cc, device=DEV, generator=g) * 0.1
    rv0 = torch.rand(Cc, device=DEV, generator=g) + 0.5
    eps, nbt0 = 1e-3, 5
    acc = _Acc(Cc)

    def run():
        o = {k: _guarded(Cc) for k in ("scale", "shift", "mean", "invstd")}
        o["rm"], o["rv"] = _guarded(Cc), _guarded(Cc)
        o["rm"][:Cc], o["rv"][:Cc] = rm0, rv0
        o["nbt"] = torch.full((1,), nbt0, device=DEV, dtype=torch.int64)
        f = nat.BnFwd()
        f.partials, f.counter = acc.partials.data_ptr(), acc.counter.data_ptr()
        f.gamma = None if gamma is None else gamma.data_ptr()
        f.beta = None if beta is None else beta.data_ptr()
        f.eps, f.momentum = eps, -1.0 if c.mom is None else c.mom
        f.running_mean, f.running_var = o["rm"].data_ptr(), o["rv"].data_ptr()
        f.num_batches_tracked = o["nbt"].data_ptr()
        f.scale, f.shift = o["scale"].data_ptr(), o["shift"].data_ptr()
        f.mean, f.invstd = o["mean"].data_ptr(), o["invstd"].data_ptr()
        f.count = M
        s = nat.BnStats()
        s.M, s.C, s.ldh, s.h, s.bn = M, Cc, ld, h.data_ptr() + 2 * c0, C.pointer(f)
        nat.check(built_lib.yamb_bn_stats_fwd(C.byref(s), nat.stream_handle()))
        acc.check()
        return o

    o = run()
    o2 = run()
    for k in o:
        _same(o[k], o2[k], "bn_stats " + k)
        if k != "nbt":
            _check_guard(o[k], Cc, "bn_stats " + k)
    loc = _chan_loc(plan)

    # the reference module itself: running statistics, num_batches_tracked
    h64 = h[:M, c0:c0 + Cc].double()
    s_ref, q_ref = h64.sum(0), (h64 * h64).sum(0)
    b_s = _long_bound(s_ref, (h64 ** 2).sum(0).sqrt())
    b_q = _long_bound(q_ref, (h64 ** 4).sum(0).sqrt())
    mean_ref, var_ref, inv_ref = _check_fwd_finalize(o, h64, gamma, beta, rm0, rv0, nbt0, eps, c.mom,
                                                     b_s, b_q, "bn_stats", loc)
    mean_got, inv_got = o["mean"][:Cc], o["invstd"][:Cc]
    if c.data == "shifted":
        ratio = float((mean_ref.abs() / var_ref.sqrt()).median())
        e_m = float(((mean_got.double() - mean_ref) / mean_ref).abs().max())
        e_i = float(((inv_got.double() - inv_ref) / inv_ref).abs().max())
        print("\nshifted statistics: median |mean|/std %.1f, max rel err mean %.2e invstd %.2e"
              % (ratio, e_m, e_i))
        assert ratio > 15.0
        assert e_m < 1e-4 and e_i < 1e-4, (e_m, e_i)


# ---- bn_reduce + bn_bwd_apply ------------------------------------------------------------------
@pytest.mark.parametrize("c", ec.BWD_CASES, ids=lambda c: "M%d-C%d-act%d-%s" % (c.M, c.C, c.act, c.why))
def test_bn_backward(built_lib, c):
    nat = _nat()
    sms = _sms()
    rplan, aplan = ec.reduce_plan(c.M, c.C, sms), ec.bwd_apply_plan(c.M, c.C, sms)
    g = torch.Generator(device=DEV).manual_seed(13)
    M, Cc, ld, c0 = c.M, c.C, c.ld, c.c0
    h = _with_poison(_bf((M, ld), 1.5, 0.3, g))
    dy = _with_poison(_bf((M, ld), 1.0, 0.0, g))
    h64, dy64 = h[:M, c0:c0 + Cc].double(), dy[:M, c0:c0 + Cc].double()
    gamma = torch.rand(Cc, device=DEV, generator=g) + 0.5 if c.affine else None
    mean1 = _f32(h64.mean(0)) if M > 1 else torch.zeros(Cc, device=DEV)
    invstd1 = _f32((h64.var(0, unbiased=False) + 1e-3).rsqrt()) if M > 1 else \
        torch.ones(Cc, device=DEV)
    zs = torch.rand(Cc, device=DEV, generator=g) + 0.5 if c.act else None
    zt = torch.randn(Cc, device=DEV, generator=g) * 0.3 if c.act else None
    z32 = _f32(h64 * zs.double() + zt.double()) if c.act else h64.float()
    gp = _dact64(z32, c.act)
    dz64 = dy64 * gp
    acc = _Acc(Cc)

    if M > 1:
        xhat = (h64 - mean1.double()) * invstd1.double()
        s_ref, q_ref = dz64.sum(0), (dz64 * xhat).sum(0)
        aerr = dy64.abs() * _act_err(z32.double(), c.act, gp)
        b_s = _long_bound(s_ref, (dz64 ** 2).sum(0).sqrt()) + aerr.sum(0)
        b_q = _long_bound(q_ref, ((dz64 * xhat) ** 2).sum(0).sqrt()) + \
            (aerr * xhat.abs()).sum(0) + 2.0 ** -22 * (dz64 * xhat).abs().sum(0)
        dg0 = (torch.randn(Cc, device=DEV, dtype=torch.float64, generator=g) *
               ((dz64 * xhat) ** 2).sum(0).sqrt()).float()
        db0 = (torch.randn(Cc, device=DEV, dtype=torch.float64, generator=g) *
               (dz64 ** 2).sum(0).sqrt()).float()

        def reduce(use_batch_stats):
            out = _bwd_outputs(Cc, dg0, db0)
            b = _bn_bwd(acc, Cc, M, gamma, mean1, invstd1, out, use_batch_stats)
            r = nat.BnReduce()
            r.M, r.C, r.lddy, r.ldh = M, Cc, ld, ld
            r.dy, r.h, r.bn = dy.data_ptr() + 2 * c0, h.data_ptr() + 2 * c0, C.pointer(b)
            if c.act:
                r.z_scale, r.z_shift, r.z_act = zs.data_ptr(), zt.data_ptr(), c.act
            nat.check(built_lib.yamb_bn_reduce_bwd(C.byref(r), nat.stream_handle()))
            acc.check()
            return out

        out = reduce(1)
        out2 = reduce(1)
        for k in out:
            _same(out[k], out2[k], "bn_reduce " + k)
        _check_bwd_finalize(out, Cc, M, gamma, mean1, invstd1, s_ref, q_ref, b_s, b_q, dg0, db0,
                            "bn_reduce", _chan_loc(rplan))
        _eval_mode_coeffs(reduce, out, Cc, gamma, invstd1, "bn_reduce")
        ca, cb, cc = out["ca"][:Cc], out["cb"][:Cc], out["cc"][:Cc]
    else:      # one row: no batch statistics to reduce; coefficients of a plausible size
        ca = torch.rand(Cc, device=DEV, generator=g) + 0.5
        cb = torch.randn(Cc, device=DEV, generator=g) * 0.2
        cc = torch.randn(Cc, device=DEV, generator=g) * 0.1

    def apply():
        dh = torch.full((M + 1, ld), SENTINEL, device=DEV, dtype=torch.bfloat16)
        a = nat.BnBwdApply()
        a.M, a.C, a.lddy, a.ldh, a.lddh = M, Cc, ld, ld, ld
        a.dy, a.h = dy.data_ptr() + 2 * c0, h.data_ptr() + 2 * c0
        if c.act:
            a.z_scale, a.z_shift, a.z_act = zs.data_ptr(), zt.data_ptr(), c.act
        a.ca, a.cb, a.cc = ca.data_ptr(), cb.data_ptr(), cc.data_ptr()
        a.dh = dh.data_ptr() + 2 * c0
        nat.check(built_lib.yamb_bn_bwd_apply_bwd(C.byref(a), nat.stream_handle()))
        torch.cuda.synchronize()
        return dh

    dh = apply()
    _same(dh, apply(), "bn_bwd_apply dh")
    _check_frame(dh, M, c0, Cc, "bn_bwd_apply")
    got = dh[:M, c0:c0 + Cc]
    loc = _walk_loc(aplan, 4)
    t1 = _f32(cb.double() * h64 + cc.double())
    if c.act in (0, 1, 2):
        d = dy64 * gp                    # dy or 0: exact
        _equal(got, _f32(ca.double() * d + t1.double()).to(torch.bfloat16), "bn_bwd_apply dh", loc)
    else:
        cad = ca.double() * dy64
        y64 = cad * gp + cb.double() * h64 + cc.double()
        delta = cad.abs() * _act_err(z32.double(), c.act, gp) + \
            2.0 ** -22 * ((cad * gp).abs() + t1.double().abs()) + \
            2.0 ** -23 * ((cb.double() * h64).abs() + cc.double().abs())
        _between(got, y64, delta, "bn_bwd_apply dh", loc)


# ---- se_pool + se_bwd_reduce -------------------------------------------------------------------
@pytest.mark.parametrize("c", ec.SE_CASES, ids=lambda c: "N%d-HW%d-C%d-%s" % (c.N, c.HW, c.C, c.why))
def test_se_pool_and_bwd_reduce(built_lib, c):
    nat = _nat()
    g = torch.Generator(device=DEV).manual_seed(14)
    N, HW, Cc, ld, c0 = c.N, c.HW, c.C, c.ld, c.c0
    M = N * HW
    h = _with_poison(_bf((M, ld), 1.5, 0.3, g))
    dy = _with_poison(_bf((M, ld), 1.0, 0.0, g))
    scale = torch.rand(Cc, device=DEV, generator=g) + 0.5
    shift = torch.randn(Cc, device=DEV, generator=g) * 0.3

    def pool():
        out = _guarded(N * Cc, SENTINEL)
        p = nat.SePool()
        p.N, p.HW, p.C, p.ldh = N, HW, Cc, ld
        p.h, p.scale, p.shift, p.act = h.data_ptr() + 2 * c0, scale.data_ptr(), shift.data_ptr(), c.act
        p.pooled = out.data_ptr()
        nat.check(built_lib.yamb_se_pool_fwd(C.byref(p), nat.stream_handle()))
        torch.cuda.synchronize()
        return out

    def dgate():
        out = _guarded(N * Cc, SENTINEL)
        r = nat.SeBwdReduce()
        r.N, r.HW, r.C, r.ldd, r.ldh = N, HW, Cc, ld, ld
        r.dy, r.h = dy.data_ptr() + 2 * c0, h.data_ptr() + 2 * c0
        r.scale, r.shift, r.act = scale.data_ptr(), shift.data_ptr(), c.act
        r.dgate = out.data_ptr()
        nat.check(built_lib.yamb_se_bwd_reduce_bwd(C.byref(r), nat.stream_handle()))
        torch.cuda.synchronize()
        return out

    pooled, dg = pool(), dgate()
    _same(pooled, pool(), "se_pool pooled")
    _same(dg, dgate(), "se_bwd_reduce dgate")
    _check_guard(pooled, N * Cc, "se_pool")
    _check_guard(dg, N * Cc, "se_bwd_reduce")

    h64 = h[:M, c0:c0 + Cc].double()
    dy64 = dy[:M, c0:c0 + Cc].double()
    z32 = _f32(h64 * scale.double() + shift.double())
    if c.act in (0, 1, 2):
        a = _clamp32(z32, c.act).to(torch.bfloat16).double()
        band = torch.zeros_like(a)
    else:
        ae = _act64(z32, c.act)
        a = ae.float().to(torch.bfloat16).double()
        band = _staged_band(ae)
    chunks = ec.se_chunks(N, HW, Cc, _sms())
    rows_per = ec.cdiv(HW, chunks)

    def loc(n, ch):
        return "(sample %d, channel %d: launch %d of 2048 channels, %d pixel chunks of %d rows)" % (
            n, ch, ch // 2048, chunks, rows_per)

    per = lambda t: t.view(N, HW, Cc).sum(1)
    p_ref = per(a) / HW
    p_b = _long_bound(p_ref, per(a * a).sqrt() / HW) + per(band) / HW
    _worst((pooled[:N * Cc].view(N, Cc).double() - p_ref).abs(), p_b, "se_pool pooled", loc)
    t = dy64 * a
    d_ref = per(t)
    d_b = _long_bound(d_ref, per(t * t).sqrt()) + per(dy64.abs() * band)
    _worst((dg[:N * Cc].view(N, Cc).double() - d_ref).abs(), d_b, "se_bwd_reduce dgate", loc)


# ---- se_bwd_apply --------------------------------------------------------------------------------
@pytest.mark.parametrize("c", ec.SE_APPLY_CASES,
                         ids=lambda c: "N%d-HW%d-C%d-of%d-%s" % (c.N, c.HW, c.C, c.Chid, c.why))
def test_se_bwd_apply(built_lib, c):
    nat = _nat()
    g = torch.Generator(device=DEV).manual_seed(15)
    N, HW, Cc, Ch, c0 = c.N, c.HW, c.C, c.Chid, c.c0
    M = N * HW
    plan = ec.se_apply_plan(M, Cc, _sms())
    h = _with_poison(_bf((M, Ch), 1.5, 0.3, g))
    dy = _with_poison(_bf((M, Ch), 1.0, 0.0, g))
    scale = torch.rand(Ch, device=DEV, generator=g) + 0.5
    shift = torch.randn(Ch, device=DEV, generator=g) * 0.3
    gate = torch.rand(N, Ch, device=DEV, generator=g)
    dpool = torch.randn(N, Ch, device=DEV, generator=g) * 0.05
    h64, dy64 = h[:M, c0:c0 + Cc].double(), dy[:M, c0:c0 + Cc].double()
    gamma = torch.rand(Cc, device=DEV, generator=g) + 0.5 if c.act != 2 else None
    mean1 = _f32(h64.mean(0))
    invstd1 = _f32((h64.var(0, unbiased=False) + 1e-3).rsqrt())
    acc = _Acc(Cc)
    rows = torch.arange(M, device=DEV) // HW
    z32 = _f32(h64 * scale[c0:c0 + Cc].double() + shift[c0:c0 + Cc].double())
    gp = _dact64(z32, c.act)
    u32 = _f32(dy64 * gate[rows, c0:c0 + Cc].double() + dpool[rows, c0:c0 + Cc].double())
    xhat = (h64 - mean1.double()) * invstd1.double()
    scale_q = (u32.double() * gp * xhat) ** 2
    dg0 = (torch.randn(Cc, device=DEV, dtype=torch.float64, generator=g) *
           scale_q.sum(0).sqrt()).float()
    db0 = (torch.randn(Cc, device=DEV, dtype=torch.float64, generator=g) *
           ((u32.double() * gp) ** 2).sum(0).sqrt()).float()

    def run(use_batch_stats=1, in_place=False):
        dyb = dy.clone()
        dz = dyb if in_place else torch.full((M + 1, Ch), SENTINEL, device=DEV, dtype=torch.bfloat16)
        out = _bwd_outputs(Cc, dg0, db0)
        b = _bn_bwd(acc, Cc, M, gamma, mean1, invstd1, out, use_batch_stats)
        a = nat.SeBwdApply()
        a.M, a.C, a.ldd, a.ldh, a.ldz, a.rows_per_sample = M, Cc, Ch, Ch, Ch, HW
        a.dy, a.h = dyb.data_ptr() + 2 * c0, h.data_ptr() + 2 * c0
        a.scale, a.shift, a.act = scale.data_ptr() + 4 * c0, shift.data_ptr() + 4 * c0, c.act
        a.gate, a.dpool, a.ldg = gate.data_ptr() + 4 * c0, dpool.data_ptr() + 4 * c0, Ch
        a.dz = dz.data_ptr() + 2 * c0
        a.bn = C.pointer(b)
        nat.check(built_lib.yamb_se_bwd_apply_bwd(C.byref(a), nat.stream_handle()))
        acc.check()
        out["dz"] = dz
        return out

    out = run()
    out2 = run()
    for k in out:
        _same(out[k], out2[k], "se_bwd_apply " + k)
    dz = out["dz"]
    _check_frame(dz, M, c0, Cc, "se_bwd_apply")
    inp = run(in_place=True)
    _same(inp["dz"][:M, c0:c0 + Cc], dz[:M, c0:c0 + Cc], "se_bwd_apply in place (dz == dy) vs out of place")
    _same(inp["dz"][:, :c0], dy[:, :c0], "se_bwd_apply in place: channels before the slice")
    _same(inp["dz"][:, c0 + Cc:], dy[:, c0 + Cc:], "se_bwd_apply in place: channels after the slice")
    for k in ("ca", "cb", "cc", "dg", "db"):
        _same(inp[k], out[k], "se_bwd_apply in place " + k)

    loc = _walk_loc(plan, 1)
    got = dz[:M, c0:c0 + Cc]
    if c.act in (0, 1, 2):
        _equal(got, (u32 * gp.float()).to(torch.bfloat16), "se_bwd_apply dz", loc)
    else:
        y64 = u32.double() * gp
        delta = u32.double().abs() * _act_err(z32.double(), c.act, gp) + 2.0 ** -22 * y64.abs()
        _between(got, y64, delta, "se_bwd_apply dz", loc)
    # statistics: of the exact dz (the issue's long-sum bound, with the bf16 rounding of the stored
    # values inside 2^-8 Q), and of the stored values at the fp32 accumulation bound
    r = got.double()
    s_ref, q_ref = r.sum(0), (r * xhat).sum(0)
    tight = 2.0 ** -24 * (plan.iters + 2)
    b_s = tight * r.abs().sum(0)
    b_q = tight * (r * xhat).abs().sum(0) + 2.0 ** -22 * (r * xhat).abs().sum(0)
    e64 = u32.double() * gp
    aerr = u32.double().abs() * _act_err(z32.double(), c.act, gp) + 2.0 ** -9 * e64.abs()
    _worst((s_ref - e64.sum(0)).abs(),
           _long_bound(e64.sum(0), (e64 ** 2).sum(0).sqrt()) + aerr.sum(0),
           "se_bwd_apply sum(dz) of the stored vs the exact values", _chan_loc(plan))
    _check_bwd_finalize(out, Cc, M, gamma, mean1, invstd1, s_ref, q_ref, b_s, b_q, dg0, db0,
                        "se_bwd_apply", _chan_loc(plan))
    _eval_mode_coeffs(lambda u: run(u), out, Cc, gamma, invstd1, "se_bwd_apply")


# ---- activation boundaries -----------------------------------------------------------------------
_EDGES = [0.0, 6.0, -3.0, 3.0]
_POINTS = _EDGES + [-6.0, -1.0, 1.0, 5.5, 6.5, -2.5, 2.5, 0.5]


@pytest.mark.parametrize("act", [1, 2, 3, 4])
def test_activation_boundaries(built_lib, act):
    """z exactly 0, 6, -3 and +3 (scale 1, shift 0, bf16-exact h): the gradients of the three
    backward kernels follow fp64 autograd through nn.ReLU / nn.ReLU6 / Swish / HSwish — 0 at both
    ReLU6 edges and at ReLU's 0, 0 at h-swish -3 and 1 at +3."""
    nat = _nat()
    g = torch.Generator(device=DEV).manual_seed(16)
    M, Cc = 64, 8
    pts = torch.tensor(_POINTS, device=DEV)
    idx = (torch.arange(M, device=DEV)[:, None] + torch.arange(Cc, device=DEV)[None, :]) % len(pts)
    h = pts[idx].to(torch.bfloat16)
    assert torch.equal(h.float(), pts[idx])
    dy = _bf((M, Cc), 1.0, 0.0, g)
    one, zero = torch.ones(Cc, device=DEV), torch.zeros(Cc, device=DEV)
    gp = _dact64(h.float(), act)
    want = dy.double() * gp
    edge = torch.zeros_like(h, dtype=torch.bool)
    for e in (_EDGES if act != 3 else [0.0]):        # Swish is smooth: its only exact point is 0
        edge |= h.float() == e
    expect = {1: {0.0: 0, 6.0: 1, -3.0: 0, 3.0: 1}, 2: {0.0: 0, 6.0: 0, -3.0: 0, 3.0: 1},
              4: {0.0: 0.5, 6.0: 1, -3.0: 0, 3.0: 1}}
    for e, v in expect.get(act, {}).items():
        assert bool((gp[h.float() == e] == v).all()), ("reference derivative", act, e)

    def check(got, what):
        got = got.double()
        _equal(got[edge], want[edge].float().to(torch.bfloat16), what + " at the edges")
        _between(got, want, dy.double().abs() * _act_err(h.double(), act, gp) +
                 2.0 ** -22 * want.abs(), what)

    # bn_bwd_apply with ca = 1, cb = cc = 0: dh = dy * act'(z)
    dh = torch.empty(M, Cc, device=DEV, dtype=torch.bfloat16)
    a = nat.BnBwdApply()
    a.M, a.C, a.lddy, a.ldh, a.lddh = M, Cc, Cc, Cc, Cc
    a.dy, a.h, a.dh = dy.data_ptr(), h.data_ptr(), dh.data_ptr()
    a.z_scale, a.z_shift, a.z_act = one.data_ptr(), zero.data_ptr(), act
    a.ca, a.cb, a.cc = one.data_ptr(), zero.data_ptr(), zero.data_ptr()
    nat.check(built_lib.yamb_bn_bwd_apply_bwd(C.byref(a), nat.stream_handle()))
    torch.cuda.synchronize()
    check(dh, "bn_bwd_apply")

    # se_bwd_apply with gate 1, dpool 0: dz = dy * act'(z); its dbeta = sum dz
    acc = _Acc(Cc)
    out = _bwd_outputs(Cc, zero, zero)
    b = _bn_bwd(acc, Cc, M, None, zero, one, out)
    dz = torch.empty(M, Cc, device=DEV, dtype=torch.bfloat16)
    gate, dpool = torch.ones(2, Cc, device=DEV), torch.zeros(2, Cc, device=DEV)
    s = nat.SeBwdApply()
    s.M, s.C, s.ldd, s.ldh, s.ldz, s.rows_per_sample = M, Cc, Cc, Cc, Cc, M // 2
    s.dy, s.h, s.dz = dy.data_ptr(), h.data_ptr(), dz.data_ptr()
    s.scale, s.shift, s.act = one.data_ptr(), zero.data_ptr(), act
    s.gate, s.dpool, s.ldg = gate.data_ptr(), dpool.data_ptr(), Cc
    s.bn = C.pointer(b)
    nat.check(built_lib.yamb_se_bwd_apply_bwd(C.byref(s), nat.stream_handle()))
    acc.check()
    check(dz, "se_bwd_apply")
    _worst((out["db"][:Cc].double() - dz.double().sum(0)).abs(),
           2.0 ** -20 * dz.double().abs().sum(0), "se_bwd_apply dbeta")

    # bn_reduce: dbeta = sum dy * act'(z)
    out = _bwd_outputs(Cc, zero, zero)
    b = _bn_bwd(acc, Cc, M, None, zero, one, out)
    r = nat.BnReduce()
    r.M, r.C, r.lddy, r.ldh = M, Cc, Cc, Cc
    r.dy, r.h, r.bn = dy.data_ptr(), h.data_ptr(), C.pointer(b)
    r.z_scale, r.z_shift, r.z_act = one.data_ptr(), zero.data_ptr(), act
    nat.check(built_lib.yamb_bn_reduce_bwd(C.byref(r), nat.stream_handle()))
    acc.check()
    s_ref = want.sum(0)
    _worst((out["db"][:Cc].double() - s_ref).abs(),
           2.0 ** -20 * want.abs().sum(0) + (dy.double().abs() * _act_err(h.double(), act, gp)).sum(0),
           "bn_reduce dbeta")


# ---- shared-memory limit -------------------------------------------------------------------------
def test_statistics_kernels_refuse_channels_beyond_shared_memory(built_lib):
    """2 * C doubles of shared memory: a C beyond the device's opt-in maximum is refused with
    YAMB_EINVAL before any launch."""
    nat = _nat()
    Cc = 16384
    h = torch.zeros(1, Cc, device=DEV, dtype=torch.bfloat16)
    v = torch.zeros(Cc, device=DEV)
    acc = _Acc(Cc)
    f = nat.BnFwd()
    f.partials, f.counter = acc.partials.data_ptr(), acc.counter.data_ptr()
    f.scale, f.shift, f.count = v.data_ptr(), v.data_ptr(), 1
    s = nat.BnStats()
    s.M, s.C, s.ldh, s.h, s.bn = 1, Cc, Cc, h.data_ptr(), C.pointer(f)
    rc = built_lib.yamb_bn_stats_fwd(C.byref(s), nat.stream_handle())
    assert rc == -1 and b"shared memory" in built_lib.yamb_last_error(), built_lib.yamb_last_error()
    out = {k: v for k in ("ca", "cb", "cc", "dg", "db")}
    b = _bn_bwd(acc, Cc, 1, None, v, v, out)
    r = nat.BnReduce()
    r.M, r.C, r.lddy, r.ldh, r.dy, r.h, r.bn = 1, Cc, Cc, Cc, h.data_ptr(), h.data_ptr(), C.pointer(b)
    rc = built_lib.yamb_bn_reduce_bwd(C.byref(r), nat.stream_handle())
    assert rc == -1 and b"shared memory" in built_lib.yamb_last_error(), built_lib.yamb_last_error()
    a = nat.SeBwdApply()
    a.M, a.C, a.ldd, a.ldh, a.ldz, a.rows_per_sample = 1, Cc, Cc, Cc, Cc, 1
    a.dy, a.h, a.dz = h.data_ptr(), h.data_ptr(), h.data_ptr()
    a.scale, a.shift, a.gate, a.dpool, a.ldg = v.data_ptr(), v.data_ptr(), v.data_ptr(), v.data_ptr(), Cc
    a.bn = C.pointer(b)
    rc = built_lib.yamb_se_bwd_apply_bwd(C.byref(a), nat.stream_handle())
    assert rc == -1 and b"shared memory" in built_lib.yamb_last_error(), built_lib.yamb_last_error()
    torch.cuda.synchronize()
