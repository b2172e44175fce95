"""GPU parity of the depthwise kernels against a float64 reference of the same op (F.conv2d /
torch.nn.grad on .double() tensors) with the kernel's bf16 staging points, element by element.

Staged operands.  The forward stages a1 = bf16(act(fp32(sc*x + sh))): fp32(...) is one fmaf, which
the reference reproduces by forming sc*x + sh in fp64 (the product of an fp32 and a bf16 value is
exact there) and rounding once to fp32.  The backward stages dh = bf16(fmaf(ca, dz, fmaf(cb, h,
cc))), reproduced the same way.  With no activation, ReLU or ReLU6 the reference operands equal the
kernel's bit for bit.  Swish and h-swish run on fast intrinsics: their staged value may sit one
bf16 ulp from the reference's wherever the exact activation lies within 2^-16 (relative) of a bf16
rounding boundary; `band` is the width of that ulp at such elements and 0 elsewhere.

Short sums (y and dx: at most k*k = 49 products per output).  With r the fp64 reference, S the sum
of the absolute products and E = conv(band, |w|),
    |got - r| <= 2^-8 |r| + 2^-16 S + E
2^-8 |r| is the rounding of the stored bf16 value, 2^-16 S covers fp32 accumulation of <= 49 terms
(and fp32 activation gradients), E the staging ulps.  A dropped or misplaced tap costs about the
largest product T >= S / 49, more than 2^5 times 2^-16 S + 2^-8 |r| wherever |r| is small.

Long sums (dw per (channel, tap); per channel sum(y), sum(y^2), sum(dx), sum(dx * xhat)): up to
N*H*W signed terms, so the value is about sqrt(n) times smaller than the sum of |terms| and a bound
that scales with the latter would hide a whole tile.  With Q = sqrt(sum term^2),
    |got - r| <= 2^-10 |r| + 2^-8 Q
A missing tile of ~100 pixels out of n ~ 1e5 changes the sum by ~Q sqrt(100 / n) = 0.03 Q: eight
times the allowance.  mean, invstd, the running statistics and ca / cb / cc are derived from these
sums in fp64 and gated with the bound propagated through that derivation (plus fp32 rounding of
the stored values); dw, dgamma and dbeta are ACCUMULATED (+=) into pre-filled buffers, whose fp32
addition adds 2^-23 (|pre| + |r|).

Besides the values, every call is checked for: channels outside the slice [c0, c0 + C) of y and dx
keep a sentinel; the BatchNorm accumulator and counter come back zero; an identical second call
from identical buffers gives identical bits; the forward without BatchNorm gives the same y; the
backward with use_batch_stats = 0 (eval-mode BatchNorm) gives cb = cc = 0, ca = gamma * invstd and
the same dx, dw, dgamma, dbeta.  The old small cases (at most one tile per CTA) keep their rel-L2
gates; the walk cases (tests/dw_cases.py) launch every instantiation with >= 2 tiles per CTA.

A CTA that changes channel chunk in the middle of its walk (flush_stats / weight reload inside the
loop) is not reached on an H100: grid_k rounds the grid down to a multiple of the chunk count, and
with <= 128 chunks and >= 132 CTAs every CTA's range starts and ends on chunk boundaries."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

import dw_cases as dc
from dw_cases import CASES, WALK_CASES

pytestmark = pytest.mark.gpu

from gpu_probe_gemm import _act, _act_grad  # noqa: E402

SENTINEL = -1536.0       # a bf16 value no output of these tests takes
BAND = 2.0 ** -16        # relative distance of an intrinsic activation from the exact one


def _rel(a, b):
    return float((a - b).norm() / (b.norm() + 1e-20))


def _nhwc(t):  # [N,C,H,W] float -> [N,H,W,C] bf16 contiguous
    return t.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)


def _nchw(t, c0, C):  # [N,H,W,ldc] bf16 slice -> [N,C,H,W] float64
    return t[..., c0:c0 + C].permute(0, 3, 1, 2).double()


def _f32(t):  # round an fp64 tensor to fp32 and back
    return t.float().double()


def _worst(err, bound, what, plan=None, c0=0):
    """Largest err / bound; on failure name the element (n, y, x, c) and its tile."""
    ratio = err / (bound + 1e-300)
    i = int(ratio.argmax())
    r = float(ratio.flatten()[i])
    if r > 1.0:
        idx = list(torch.unravel_index(torch.tensor(i), ratio.shape))
        msg = "%s: err/bound %.3g at " % (what, r)
        if ratio.dim() == 4:
            n, c, y, x = (int(v) for v in idx)
            msg += "(n=%d, y=%d, x=%d, c=%d)" % (n, y, x, c + c0)
            if plan is not None:
                msg += " tile (chunk %d, ty %d, tx %d)" % (c // plan.ct, y // plan.tile_h,
                                                           x // plan.tile_w)
        else:
            msg += str(tuple(int(v) for v in idx))
        msg += " got-ref %.4g bound %.4g" % (float(err.flatten()[i]), float(bound.flatten()[i]))
        raise AssertionError(msg)
    return r


def _long_bound(r, q):
    return 2.0 ** -10 * r.abs() + 2.0 ** -8 * q


def _staged_band(a):
    """Width of the bf16 rounding ambiguity of an activation value computed with ~2^-20 relative
    error: the bf16 values of a * (1 -+ 2^-16) differ only near a rounding boundary."""
    lo = (a * (1 - BAND)).to(torch.bfloat16).double()
    hi = (a * (1 + BAND)).to(torch.bfloat16).double()
    return (hi - lo).abs()


def _check_zero(partials, counter):
    assert int(counter.item()) == 0, "counter not returned to 0"
    assert float(partials.abs().max()) == 0.0, "BatchNorm accumulator not returned to 0"


def _same(a, b, what):
    assert torch.equal(a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8)), \
        "%s: bits differ" % what


def _run(lib, N, H, W, Ct, c0, Cs, k, s, act, pro, *, mom=-1.0, nbt0=0, prefill=False,
         x=None, w=None, seed=1):
    """One forward + backward of the depthwise stage, every check of the module docstring.
    Returns the worst err / bound ratios and the launch plans."""
    from yet_another_mobilenet_series_b200 import native as nat
    dev = "cuda"
    torch.manual_seed(seed)
    pad = (k - 1) // 2
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    fplan, bplan = dc.fwd_plan(N, H, W, Cs, k, s), dc.bwd_plan(N, H, W, Cs, k, s)
    if x is None:
        x = torch.randn(N, Ct, H, W, device=dev)
    xb = _nhwc(x)
    x64 = _nchw(xb, c0, Cs)
    if w is None:
        w = torch.randn(Cs, 1, k, k, device=dev) * 0.3
    w64 = w.double()
    sc = torch.rand(Cs, device=dev) + 0.5
    sh = torch.randn(Cs, device=dev) * 0.3
    v = lambda t: t.double()[None, :, None, None]
    bn_acc = torch.zeros(2 * Cs + 64, device=dev, dtype=torch.float64)   # + guard
    counter = torch.zeros(1, device=dev, dtype=torch.int32)
    worst = {}

    # ---------------- reference forward ----------------
    # the kernel stages act(fmaf(sc, x, sh)) in shared memory as bf16
    if pro:
        z64 = _f32(x64 * v(sc) + v(sh))
        a_exact = _act(z64, act)
        a1 = a_exact.to(torch.bfloat16).double()
        band = _staged_band(a_exact) if act in (3, 4) else None
    else:
        z64, a1, band = None, x64, None
    y64 = F.conv2d(a1, w64, None, s, pad, 1, Cs)
    y_sabs = F.conv2d(a1.abs(), w64.abs(), None, s, pad, 1, Cs)
    y_bound = 2.0 ** -8 * y64.abs() + 2.0 ** -16 * y_sabs
    if band is not None:
        y_bound += F.conv2d(band, w64.abs(), None, s, pad, 1, Cs)

    # ---------------- forward ----------------
    gamma = torch.rand(Cs, device=dev) + 0.5
    beta = torch.randn(Cs, device=dev)
    rm0 = torch.randn(Cs, device=dev) * 0.1
    rv0 = torch.rand(Cs, device=dev) + 0.5
    eps = 1e-3

    def fwd(with_bn):
        st = dict(y=torch.full((N, Ho, Wo, Ct), SENTINEL, device=dev, dtype=torch.bfloat16),
                  rm=rm0.clone(), rv=rv0.clone(),
                  nbt=torch.full((1,), nbt0, device=dev, dtype=torch.int64),
                  scale=torch.zeros(Cs, device=dev), shift=torch.zeros(Cs, device=dev),
                  mean=torch.zeros(Cs, device=dev), invstd=torch.zeros(Cs, device=dev))
        bn = nat.BnFwd()
        bn.partials, bn.counter = bn_acc.data_ptr(), counter.data_ptr()
        bn.gamma, bn.beta, bn.eps, bn.momentum = gamma.data_ptr(), beta.data_ptr(), eps, mom
        bn.running_mean, bn.running_var = st["rm"].data_ptr(), st["rv"].data_ptr()
        bn.num_batches_tracked = st["nbt"].data_ptr()
        bn.scale, bn.shift = st["scale"].data_ptr(), st["shift"].data_ptr()
        bn.mean, bn.invstd = st["mean"].data_ptr(), st["invstd"].data_ptr()
        bn.count = N * Ho * Wo
        d = nat.DwFwd()
        d.N, d.H, d.W, d.C, d.ldc, d.k, d.stride = N, H, W, Cs, Ct, k, s
        d.x = xb.data_ptr() + c0 * 2
        if pro:
            d.in_scale, d.in_shift, d.in_act = sc.data_ptr(), sh.data_ptr(), act
        d.w, d.y = w.data_ptr(), st["y"].data_ptr() + c0 * 2
        if with_bn:
            d.bn = C.pointer(bn)
        nat.check(lib.yamb_depthwise_fwd(C.byref(d), nat.stream_handle()))
        torch.cuda.synchronize()
        _check_zero(bn_acc, counter)
        return st

    f1 = fwd(True)
    yb = f1["y"]
    y_got = _nchw(yb, c0, Cs)
    worst["y"] = _worst((y_got - y64).abs(), y_bound, "y", fplan, c0)
    assert _rel(y_got, y64.to(torch.bfloat16).double()) < 4e-3
    assert bool((yb[..., :c0] == SENTINEL).all()) and bool((yb[..., c0 + Cs:] == SENTINEL).all()), \
        "forward wrote channels outside [c0, c0 + C)"
    f2 = fwd(True)
    for key in f1:
        _same(f1[key], f2[key], "forward " + key)
    f3 = fwd(False)   # eval-mode forward: no statistics, the same y, nothing else written
    _same(f1["y"], f3["y"], "y without BatchNorm")
    assert torch.equal(f3["rm"], rm0) and torch.equal(f3["rv"], rv0) and int(f3["nbt"]) == nbt0
    assert float(f3["mean"].abs().max()) == 0.0 and float(f3["scale"].abs().max()) == 0.0

    # statistics come from the fp32 accumulators (before the bf16 rounding of the stored tensor)
    cnt = N * Ho * Wo
    red = lambda t: t.sum((0, 2, 3))
    s_ref, q_ref = red(y64), red(y64 * y64)
    b_s = _long_bound(s_ref, red(y64 ** 2).sqrt())
    b_q = _long_bound(q_ref, red(y64 ** 4).sqrt())
    mean_ref = s_ref / cnt
    var_ref = red((y64 - v(mean_ref)) ** 2) / cnt
    e_mean = b_s / cnt
    e_var = b_q / cnt + 2 * mean_ref.abs() * e_mean + e_mean ** 2
    inv_ref = (var_ref + eps).rsqrt()
    lo = (var_ref + eps - e_var).clamp_min(1e-300)
    e_inv = 0.5 * e_var * lo ** -1.5 + 2.0 ** -23 * inv_ref
    st = {}
    st["mean"] = _worst((f1["mean"].double() - mean_ref).abs(),
                        e_mean + 2.0 ** -23 * mean_ref.abs(), "mean")
    st["invstd"] = _worst((f1["invstd"].double() - inv_ref).abs(), e_inv, "invstd")
    assert _rel(f1["mean"].double(), mean_ref) < 1e-3
    assert _rel(f1["invstd"].double(), inv_ref) < 1e-3
    # scale / shift from the stored mean / invstd in fp32
    scl = gamma * f1["invstd"]
    assert torch.equal(f1["scale"], scl)
    st["shift"] = _worst((f1["shift"].double() - (beta.double() - f1["mean"].double() * scl.double())).abs(),
                         2.0 ** -22 * (beta.double().abs() + (f1["mean"] * scl).double().abs()), "shift")
    # running statistics, nn.BatchNorm2d semantics: unbiased variance, momentum or 1/(nbt+1)
    fac = torch.tensor(mom if mom >= 0 else 1.0, dtype=torch.float32)
    if mom < 0:
        fac = fac / float(nbt0 + 1)
    fac = float(fac)
    one_m = float(torch.tensor(1.0, dtype=torch.float32) - torch.tensor(fac, dtype=torch.float32))
    unb = cnt / (cnt - 1)
    rm_ref = one_m * rm0.double() + fac * mean_ref
    rv_ref = one_m * rv0.double() + fac * var_ref * unb
    rnd = lambda a, b: 2.0 ** -22 * (one_m * a.abs() + fac * b.abs())
    st["running_mean"] = _worst((f1["rm"].double() - rm_ref).abs(),
                                fac * e_mean + rnd(rm0.double(), mean_ref), "running_mean")
    st["running_var"] = _worst((f1["rv"].double() - rv_ref).abs(),
                               fac * e_var * unb + rnd(rv0.double(), var_ref * unb), "running_var")
    assert int(f1["nbt"]) == nbt0 + 1

    # ---------------- reference backward ----------------
    dz = torch.randn(N, Ct, Ho, Wo, device=dev)
    h = torch.randn(N, Ct, Ho, Wo, device=dev)
    dzb, hb = _nhwc(dz), _nhwc(h)
    ca = torch.rand(Cs, device=dev) + 0.5
    cb = torch.randn(Cs, device=dev) * 0.2
    cc = torch.randn(Cs, device=dev) * 0.1
    mean1 = torch.randn(Cs, device=dev) * 0.1
    invstd1 = torch.rand(Cs, device=dev) + 0.5
    g1 = torch.rand(Cs, device=dev) + 0.5
    res = None if pro else _nhwc(torch.randn(N, Ct, H, W, device=dev))
    dz64, h64 = _nchw(dzb, c0, Cs), _nchw(hb, c0, Cs)
    t1 = _f32(v(cb) * h64 + v(cc))
    dh = _f32(v(ca) * dz64 + t1).to(torch.bfloat16).double()     # staged as bf16
    da = torch.nn.grad.conv2d_input(a1.shape, w64, dh, s, pad, 1, Cs)
    da_sabs = torch.nn.grad.conv2d_input(a1.shape, w64.abs(), dh.abs(), s, pad, 1, Cs)
    dw_ref = torch.nn.grad.conv2d_weight(a1, w.shape, dh, s, pad, 1, Cs)
    dw_q = torch.nn.grad.conv2d_weight(a1 * a1, w.shape, dh * dh, s, pad, 1, Cs).sqrt()
    if pro:
        g = _act_grad(z64, act)
        # Swish' on intrinsics is off by ~2^-18 (1 + |z|) absolute, also where act' crosses 0
        dx_ref, dx_sabs = da * g, da_sabs * (g.abs() + (0.25 if act == 3 else 0.0))
    else:
        r64 = _nchw(res, c0, Cs)
        dx_ref, dx_sabs = da + r64, da_sabs + r64.abs()

    # BatchNorm-backward sums are taken from the fp32 gradients (before the bf16 rounding of the
    # stored dx), like the forward statistics; the kernel's xhat = fmaf(x, r, fp32(-mu*r))
    xhat = (x64 - v(mean1)) * v(invstd1)
    s_ref, q_ref = red(dx_ref), red(dx_ref * xhat)
    s_q, q_q = red(dx_ref ** 2).sqrt(), red((dx_ref * xhat) ** 2).sqrt()

    # ---------------- backward ----------------
    # dw, dgamma and dbeta are accumulated: pre-fill them with values of the size of the sums'
    # own scale Q, far outside the 2^-8 Q allowance
    pre = lambda q: ((torch.randn(q.shape, device=dev, dtype=torch.float64) * q).float()
                     if prefill else torch.zeros(q.shape, device=dev))
    dw0, dg0, db0 = pre(dw_q), pre(q_q), pre(s_q)

    def bwd(use_batch_stats):
        st = dict(dx=torch.full((N, H, W, Ct), SENTINEL, device=dev, dtype=torch.bfloat16),
                  dw=dw0.clone(), dg=dg0.clone(), db=db0.clone(),
                  ca=torch.zeros(Cs, device=dev), cb=torch.zeros(Cs, device=dev),
                  cc=torch.zeros(Cs, device=dev))
        bb = nat.BnBwd()
        bb.partials, bb.counter = bn_acc.data_ptr(), counter.data_ptr()
        bb.gamma, bb.mean, bb.invstd = g1.data_ptr(), mean1.data_ptr(), invstd1.data_ptr()
        bb.dgamma, bb.dbeta = st["dg"].data_ptr(), st["db"].data_ptr()
        bb.ca, bb.cb, bb.cc = st["ca"].data_ptr(), st["cb"].data_ptr(), st["cc"].data_ptr()
        bb.count = N * H * W
        bb.use_batch_stats = use_batch_stats
        e = nat.DwBwd()
        e.N, e.H, e.W, e.C, e.ldc, e.k, e.stride = N, H, W, Cs, Ct, k, s
        e.dz, e.h = dzb.data_ptr() + c0 * 2, hb.data_ptr() + c0 * 2
        e.ca, e.cb, e.cc = ca.data_ptr(), cb.data_ptr(), cc.data_ptr()
        e.w, e.dw = w.data_ptr(), st["dw"].data_ptr()
        e.x = xb.data_ptr() + c0 * 2
        if pro:
            e.in_scale, e.in_shift, e.in_act = sc.data_ptr(), sh.data_ptr(), act
            e.bn = C.pointer(bb)
        else:
            e.residual = res.data_ptr() + c0 * 2
        e.dx = st["dx"].data_ptr() + c0 * 2
        nat.check(lib.yamb_depthwise_bwd(C.byref(e), nat.stream_handle()))
        torch.cuda.synchronize()
        _check_zero(bn_acc, counter)
        return st

    b1 = bwd(1)
    dxb = b1["dx"]
    dx_got = _nchw(dxb, c0, Cs)
    worst["dx"] = _worst((dx_got - dx_ref).abs(),
                         2.0 ** -8 * dx_ref.abs() + 2.0 ** -16 * dx_sabs, "dx", bplan, c0)
    assert _rel(dx_got, dx_ref.to(torch.bfloat16).double()) < 4e-3
    assert bool((dxb[..., :c0] == SENTINEL).all()) and \
        bool((dxb[..., c0 + Cs:] == SENTINEL).all()), "backward wrote channels outside [c0, c0 + C)"
    dw_got = b1["dw"].double()
    worst["dw"] = _worst((dw_got - dw0.double() - dw_ref).abs().view(Cs, k * k),
                         (_long_bound(dw_ref, dw_q) +
                          2.0 ** -23 * (dw0.double().abs() + dw_ref.abs())).view(Cs, k * k),
                         "dw (channel, tap)")
    assert _rel(dw_got - dw0.double(), dw_ref) < 1e-3
    b2 = bwd(1)
    for key in b1:
        _same(b1[key], b2[key], "backward " + key)
    if pro:
        sys_q = 2.0 ** -22 * (mean1 * invstd1).double().abs() * red(dx_ref.abs())
        b_s = _long_bound(s_ref, s_q)
        b_q = _long_bound(q_ref, q_q) + sys_q
        acc = lambda p, r: 2.0 ** -23 * (p.double().abs() + r.abs())
        st["dbeta"] = _worst((b1["db"].double() - db0.double() - s_ref).abs(),
                             b_s + acc(db0, s_ref), "dbeta")
        st["dgamma"] = _worst((b1["dg"].double() - dg0.double() - q_ref).abs(),
                              b_q + acc(dg0, q_ref), "dgamma")
        assert _rel(b1["db"].double() - db0.double(), s_ref) < 2e-3
        assert _rel(b1["dg"].double() - dg0.double(), q_ref) < 2e-3
        M = N * H * W
        scl = g1 * invstd1
        assert torch.equal(b1["ca"], scl)
        sr = scl.double() * invstd1.double()
        m1, m2 = s_ref / M, q_ref / M
        cb_ref = -sr * m2
        cc_ref = scl.double() * (mean1.double() * invstd1.double() * m2 - m1)
        st["cb"] = _worst((b1["cb"].double() - cb_ref).abs(),
                          sr.abs() * b_q / M + 2.0 ** -21 * cb_ref.abs() + 1e-30, "cb")
        st["cc"] = _worst((b1["cc"].double() - cc_ref).abs(),
                          scl.double().abs() * ((mean1 * invstd1).double().abs() * b_q / M + b_s / M)
                          + 2.0 ** -21 * scl.double().abs() *
                          ((mean1 * invstd1).double().abs() * m2.abs() + m1.abs()), "cc")
        assert _rel(b1["cb"].double(), cb_ref) < 2e-3
        assert _rel(b1["cc"].double(), cc_ref) < 2e-3
        # gradients through an eval-mode BatchNorm: dh = ca * dz
        b3 = bwd(0)
        for key in ("dx", "dw", "dg", "db", "ca"):
            _same(b1[key], b3[key], "backward with use_batch_stats=0: " + key)
        assert float(b3["cb"].abs().max()) == 0.0 and float(b3["cc"].abs().max()) == 0.0
    worst["stats"] = max(st.values())
    return worst, fplan, bplan


def _report(name, lib, fplan, bplan, worst):
    nct = lib.yamb_max_ctas()
    print("\n%-34s fwd k%d s%d ct%-2d tw%d >=%5.2f tiles/CTA | bwd k%d s%d ct%-2d >=%5.2f tiles/CTA | "
          "err/bound y %.3f dx %.3f dw %.2e stats %.2e" %
          (name, *fplan.inst, fplan.num_tiles / nct, *bplan.inst, bplan.num_tiles / nct,
           worst["y"], worst["dx"], worst["dw"], worst["stats"]))


@pytest.mark.parametrize("N,H,W,Ct,c0,Cs,k,s,act,pro", CASES)
def test_depthwise_fwd_bwd(built_lib, N, H, W, Ct, c0, Cs, k, s, act, pro):
    worst, fp, bp = _run(built_lib, N, H, W, Ct, c0, Cs, k, s, act, pro)
    _report("small %dx%dx%dx%d" % (N, H, W, Cs), built_lib, fp, bp, worst)


def _walk_id(c):
    f, b = dc.fwd_plan(c.N, c.H, c.W, c.C, c.k, c.s), dc.bwd_plan(c.N, c.H, c.W, c.C, c.k, c.s)
    return "fwd%d.%d.%d.%d-bwd%d.%d.%d" % (*f.inst, *b.inst)


@pytest.mark.parametrize("case", WALK_CASES, ids=_walk_id)
def test_depthwise_walk(built_lib, case):
    c = case
    nct = built_lib.yamb_max_ctas()
    fp, bp = dc.fwd_plan(c.N, c.H, c.W, c.C, c.k, c.s), dc.bwd_plan(c.N, c.H, c.W, c.C, c.k, c.s)
    assert fp.num_tiles >= 2 * nct and bp.num_tiles >= 2 * nct, "not a walk on this device"
    worst, fp, bp = _run(built_lib, c.N, c.H, c.W, c.ldc, c.c0, c.C, c.k, c.s, c.act, c.pro,
                         mom=c.mom, nbt0=5, prefill=True, seed=2)
    _report(_walk_id(c), built_lib, fp, bp, worst)


def test_depthwise_stats_shifted(built_lib):
    """BatchNorm statistics of an output whose per-channel mean is ~20x its standard deviation:
    the kernel sums y and y^2 per thread in fp32 over every tile it walks, then in double, and
    takes var = E[y^2] - mean^2.  mean and invstd must match fp64 to 1e-4 relative."""
    from yet_another_mobilenet_series_b200 import native as nat
    lib = built_lib
    N, H, W, Cs, k = 38, 56, 56, 64, 3
    fp = dc.fwd_plan(N, H, W, Cs, k, 1)
    assert fp.num_tiles >= 2 * lib.yamb_max_ctas()
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(3)
    w = torch.rand(Cs, 1, k, k, device=dev, generator=g) + 0.5
    # input mean chosen so that the interior outputs have mean = 20 x std
    ratio = w.sum((1, 2, 3)) / w.flatten(1).norm(dim=1)
    mu = 20.0 / ratio * (1 + 0.25 * torch.rand(Cs, device=dev, generator=g))
    x = mu[None, :, None, None] + torch.randn(N, Cs, H, W, device=dev, generator=g)
    xb = _nhwc(x)
    y64 = F.conv2d(_nchw(xb, 0, Cs), w.double(), None, 1, 1, 1, Cs)
    mean_ref = y64.mean((0, 2, 3))
    var_ref = y64.var((0, 2, 3), unbiased=False)
    eps = 1e-3
    yb = torch.empty(N, H, W, Cs, device=dev, dtype=torch.bfloat16)
    acc = torch.zeros(2 * Cs, device=dev, dtype=torch.float64)
    counter = torch.zeros(1, device=dev, dtype=torch.int32)
    o = [torch.zeros(Cs, device=dev) for _ in range(4)]
    bn = nat.BnFwd()
    bn.partials, bn.counter, bn.eps, bn.momentum = acc.data_ptr(), counter.data_ptr(), eps, 0.1
    bn.scale, bn.shift, bn.mean, bn.invstd = (t.data_ptr() for t in o)
    bn.count = N * H * W
    d = nat.DwFwd()
    d.N, d.H, d.W, d.C, d.ldc, d.k, d.stride = N, H, W, Cs, Cs, k, 1
    d.x, d.w, d.y, d.bn = xb.data_ptr(), w.data_ptr(), yb.data_ptr(), C.pointer(bn)
    nat.check(lib.yamb_depthwise_fwd(C.byref(d), nat.stream_handle()))
    torch.cuda.synchronize()
    _check_zero(acc, counter)
    inv_ref = (var_ref + eps).rsqrt()
    shift = float((mean_ref / var_ref.sqrt()).median())
    e_mean = float(((o[2].double() - mean_ref) / mean_ref).abs().max())
    e_inv = float(((o[3].double() - inv_ref) / inv_ref).abs().max())
    print("\nshifted statistics: median mean/std %.1f, max rel err mean %.2e invstd %.2e"
          % (shift, e_mean, e_inv))
    assert shift > 10.0
    assert e_mean < 1e-4 and e_inv < 1e-4, (e_mean, e_inv)
