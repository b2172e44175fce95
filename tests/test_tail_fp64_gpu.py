"""GPU: the kernels at the two ends of a training step, called directly for every case of
tests/tail_cases.py and compared with a float64 reference of the same operation on the same bf16
inputs, element by element: the stem convolution (forward, eval forward, weight gradient), the
label-smoothed softmax cross entropy with top-k (forward, backward with the bias gradient) and the
bf16 column sum.  u = 2^-24 below.

Stem forward.  X27 [N*Ho*Wo, 27] is the zero-padded stride-2 unfold of x in fp64, columns in the
parameter's (ci, ky, kx) order; y64 = X27 @ W^T, A = |X27| @ |W|^T.  A bf16 x fp32 product is
exact in fp32's fma, so each of the 27 fmas rounds once by at most u A: y lies between the bf16
values of y64 -+ 27 u A.  x carries one more image of POISON after the N the kernel is given (a
halo read past the last image is far off), y a SENTINEL tail.
Stem eval.  y = bf16(act(fmaf(scale, h, shift))) with h the training forward's stored y: the
fp32 value z is the fp64 sum rounded once; no activation, ReLU and ReLU6 must match exactly,
Swish and h-swish (fp32 intrinsics) lie within BAND |a| + 2^-22 |a| of the fp64 activation.
Stem weight gradient.  dw += dh^T @ X27 onto non-zero values: |got - (dw0 + r)| <=
_long_bound(r, Q) + 2^-23 (|dw0| + |r|), Q = sqrt((dh^2)^T @ X27^2).  A walk that loses its last
tile (57 pixels of 873k) moves every element by about 0.8 % of Q; the bound is about 0.4 %.

Softmax cross entropy forward.  The kernel's operations, row by row, and the error each adds:
  x_c = fp32(v_c - mx)                     u |x_c|
  e_c = __expf(x_c)                        (2 + 1.173 |x_c|) ulp (CUDA programming guide,
                                           intrinsic functions), ulp <= 2^-23 e_c; flushed
                                           results: 2^-126 absolute
  se = sum e_c                             a chain of ceil(C/32) lane adds + 5 shuffle adds, each
                                           rounding by u of a partial sum <= se
  lse = mx + __logf(se)                    2^-21.41 absolute for se in [0.5, 2], 3 ulp otherwise
                                           (both are counted), u |lse| for the add; a relative
                                           error d of se moves it by at most 1.01 d
  sl = sum v_c                             (ceil(C/32) + 5) u sum |v|
  loss = -(1-eps)(v_t - lse) - (eps/C)(sl - C lse), each operation rounding once by u.
  G = bf16(__expf(v - lse) - eps/C - (1-eps)[c = t]): the exp's input carries |x| u and the
  error of lse; the two subtractions round by u each; G must lie between the bf16 values of
  G64 -+ that bound.
Top-1 / top-5 must equal the rank of the target in a stable descending torch.sort (lower index
first on ties), exactly; planted rows tie the target with another class at rank 1 and at ranks
5 / 6, above and below it in index, and rows at |logits| ~ 100 overflow exp without the max.
Backward.  dlogits = (G * dloss) rounded to fp32 then bf16: the fp64 product of a bf16 and an fp32
value is exact, so the stored bits must equal (G.double() * dloss.double()).float().bfloat16().
dbias += the column sums of the stored dlogits, the column sum += those of X, both under
_long_bound plus the fp32 add onto the non-zero initial values.

Every entry point: two calls give the same bits; SENTINEL survives in pitch padding, in the row
after N and in guard values; a refused call (YAMB_EINVAL) writes nothing.  On failure the message
names the element and where the launch plan put it."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

import tail_cases as tc
from ref64 import (BAND, DEV, POISON, SENTINEL, _act64, _between, _check_guard, _clamp32, _equal,
                   _f32, _guarded, _long_bound, _nat, _same, _worst)

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
U = 2.0 ** -24


def _stream():
    return _nat().stream_handle()


def _run(fn, args):
    _nat().check(fn(C.byref(args), _stream()))
    torch.cuda.synchronize()


# ---- stem ------------------------------------------------------------------------------------------
class _StemData:
    """x [N+1, H, W, 3] bf16 (image N is POISON), X27 fp64 and its absolute value."""

    def __init__(self, N, H, W):
        g = torch.Generator(device=DEV).manual_seed(N * 1009 + H * 31 + W)
        self.N, self.H, self.W = N, H, W
        self.plan = tc.stem_plan(N, H, W)
        self.xbuf = torch.full((N + 1, H, W, 3), POISON, device=DEV, dtype=BF)
        self.xbuf[:N] = torch.randn(N, H, W, 3, device=DEV, generator=g).to(BF)
        x64 = self.xbuf[:N].double().permute(0, 3, 1, 2)
        cols = F.unfold(x64, 3, padding=1, stride=2)                     # [N, 27, Ho*Wo]
        self.X27 = cols.transpose(1, 2).reshape(-1, 27).contiguous()
        del cols
        self.gen = g


_STEM = {}


def _stem_data(N, H, W):
    if (N, H, W) not in _STEM:
        if len(_STEM) > 1:
            _STEM.clear()
        _STEM[(N, H, W)] = _StemData(N, H, W)
    return _STEM[(N, H, W)]


def _stem_args(d, Cout, w=None, y=None, dh=None, dw=None):
    nat = _nat()
    a = nat.StemConv()
    a.N, a.H, a.W, a.Cout = d.N, d.H, d.W, Cout
    a.x = d.xbuf.data_ptr()
    a.w, a.y, a.dh, a.dw = (nat.ptr(t) for t in (w, y, dh, dw))
    return a


def _stem_loc(plan):
    def loc(n, oy, ox, *_):
        t = (n * plan.tiles_h + oy // tc.STEM_TH) * plan.tiles_w + ox // tc.STEM_TW
        return "(image %d, tile row %d of %d, tile column %d of %d: tile %d of %d)" % (
            n, oy // tc.STEM_TH, plan.tiles_h, ox // tc.STEM_TW, plan.tiles_w, t, plan.num_tiles)
    return loc


def _stem_fwd(lib, d, Cout, w):
    p = d.plan
    n = d.N * p.Ho * p.Wo * Cout
    buf = _guarded(n, SENTINEL, BF)
    _run(lib.yamb_stem_conv_fwd, _stem_args(d, Cout, w=w, y=buf))
    _check_guard(buf, n, "stem fwd y")
    return buf


def _check_stem_fwd(lib, c):
    d = _stem_data(c.N, c.H, c.W)
    p = d.plan
    w = torch.randn(c.Cout, 3, 3, 3, device=DEV, generator=d.gen) * 0.3
    buf = _stem_fwd(lib, d, c.Cout, w)
    _same(buf, _stem_fwd(lib, d, c.Cout, w), "stem fwd y")
    W27 = w.double().view(c.Cout, 27)
    y64 = (d.X27 @ W27.t()).view(c.N, p.Ho, p.Wo, c.Cout)
    A = (d.X27.abs() @ W27.abs().t()).view(c.N, p.Ho, p.Wo, c.Cout)
    y = buf[:c.N * p.Ho * p.Wo * c.Cout].view(c.N, p.Ho, p.Wo, c.Cout)
    _between(y, y64, 27 * U * A, "stem fwd y %s" % (tuple(c),), _stem_loc(p))
    return w, y


def _check_stem_wgrad(lib, c):
    d = _stem_data(c.N, c.H, c.W)
    p = d.plan
    g = d.gen
    dhbuf = torch.full((c.N + 1, p.Ho, p.Wo, c.Cout), POISON, device=DEV, dtype=BF)
    dhbuf[:c.N] = torch.randn(c.N, p.Ho, p.Wo, c.Cout, device=DEV, generator=g).to(BF)
    n = c.Cout * 27
    dw0 = torch.randn(n, device=DEV, generator=g)

    def run():
        dw = _guarded(n)
        dw[:n] = dw0
        _run(lib.yamb_stem_conv_wgrad, _stem_args(d, c.Cout, dh=dhbuf, dw=dw))
        _check_guard(dw, n, "stem wgrad dw")
        return dw

    dw = run()
    _same(dw, run(), "stem wgrad dw")
    dh64 = dhbuf[:c.N].double().view(-1, c.Cout)
    r = dh64.t() @ d.X27                                              # [Cout, 27]
    q = ((dh64 * dh64).t() @ (d.X27 * d.X27)).sqrt()
    got = dw[:n].double().view(c.Cout, 27)
    b0 = dw0.double().view(c.Cout, 27)
    err = (got - b0 - r).abs()
    bound = _long_bound(r, q) + 2.0 ** -23 * (b0.abs() + r.abs())

    def loc(co, j):
        return "(co %d, ci %d, ky %d, kx %d; %d tiles, %d pixels)" % (
            co, j // 9, (j % 9) // 3, j % 3, p.num_tiles, c.N * p.Ho * p.Wo)
    return _worst(err, bound, "stem wgrad dw %s" % (tuple(c),), loc)


@pytest.mark.parametrize("c", tc.STEM_CASES, ids=lambda c: "N%d-%dx%d-co%d" % c)
def test_stem_direct(built_lib, c):
    _check_stem_fwd(built_lib, c)
    if c.Cout in tc.STEM_WGRAD_COUT:
        _check_stem_wgrad(built_lib, c)


@pytest.mark.parametrize("c", tc.STEM_WALK_CASES, ids=lambda c: "N%d-%dx%d-co%d" % c)
def test_stem_walk(built_lib, c):
    plan = tc.stem_plan(c.N, c.H, c.W)
    assert tc.stem_is_walk(plan, torch.cuda.get_device_properties(0).multi_processor_count), plan
    _check_stem_fwd(built_lib, c)
    r = _check_stem_wgrad(built_lib, c)
    print("stem walk %s: wgrad err/bound %.3g" % (tuple(c), r))


@pytest.mark.parametrize("cout", tc.STEM_EVAL_COUT)
@pytest.mark.parametrize("shape", tc.STEM_EVAL_SHAPES, ids=lambda s: "N%d-%dx%d" % s)
def test_stem_eval(built_lib, shape, cout):
    nat = _nat()
    c = tc.StemCase(*shape, cout)
    d = _stem_data(*shape)
    p = d.plan
    w, h = _check_stem_fwd(built_lib, c)
    n = c.N * p.Ho * p.Wo * cout
    g = torch.Generator(device=DEV).manual_seed(cout)
    for act in range(5):
        scale = torch.rand(cout, device=DEV, generator=g) + 0.5
        shift = torch.randn(cout, device=DEV, generator=g) * 0.3

        def run():
            buf = _guarded(n, SENTINEL, BF)
            e = nat.StemConvEval()
            e.conv = _stem_args(d, cout, w=w, y=buf)
            e.scale, e.shift, e.act = scale.data_ptr(), shift.data_ptr(), act
            _run(built_lib.yamb_stem_conv_eval_fwd, e)
            _check_guard(buf, n, "stem eval y")
            return buf

        buf = run()
        _same(buf, run(), "stem eval y")
        y = buf[:n].view_as(h)
        z32 = _f32(h.double() * scale.double() + shift.double())
        what = "stem eval y %s act %d" % (tuple(c), act)
        if act in (0, 1, 2):
            _equal(y, _clamp32(z32, act).to(BF), what, _stem_loc(p))
        else:
            a64 = _act64(z32, act)
            _between(y, a64, (BAND + 2.0 ** -22) * a64.abs(), what, _stem_loc(p))


# ---- softmax cross entropy -------------------------------------------------------------------------
def _plant(v, t, C, g):
    """Rows 0..6 (where N and C allow): ties at rank 1 and at ranks 5 / 6 above and below the
    target in index, |logits| ~ 100 of both signs, an all-equal row."""
    N = v.shape[0]
    v.clamp_(-15, 15)
    rows = []
    if C >= 3:
        ti = C // 2
        rows += [(ti, ti + 1, 1), (ti, ti - 1, 1)]             # tied for the top, other after / before
    if C >= 7:
        ti = C // 2
        rows += [(ti, ti + 1, 5), (ti, ti - 1, 5)]             # tied at ranks 5 and 6
    r = 0
    for ti, other, rank in rows:
        if r >= N:
            return
        v[r, ti] = v[r, other] = 20.0
        if rank == 5:
            above = [k for k in range(C) if k not in (ti, other)][:4]
            for i, k in enumerate(above):
                v[r, k] = 30.0 + i
        t[r] = ti
        r += 1
    for sign in (1.0, -1.0):
        if r < N:
            v[r] = sign * 100.0 + 2.0 * torch.randn(C, device=DEV, generator=g)
            r += 1
    if r < N:
        v[r] = 0.25


def _ce_data(c):
    g = torch.Generator(device=DEV).manual_seed(c.N * 7919 + c.C)
    v = torch.randn(c.N, c.C, device=DEV, generator=g) * 3
    t = torch.randint(0, c.C, (c.N,), device=DEV, generator=g)
    _plant(v, t, c.C, g)
    logits = torch.full((c.N + 1, c.ld), POISON, device=DEV, dtype=BF)
    logits[:c.N, :c.C] = v.to(BF)
    return logits, t, g


def _ce_fwd(lib, c, logits, t, with_g=True, with_topk=True):
    nat = _nat()
    out = {"loss": _guarded(c.N, SENTINEL), "c1": _guarded(c.N, SENTINEL),
           "c5": _guarded(c.N, SENTINEL),
           "G": torch.full((c.N + 1, c.ldg), SENTINEL, device=DEV, dtype=BF)}
    a = nat.SoftmaxCe()
    a.N, a.C, a.ld, a.smoothing = c.N, c.C, c.ld, c.eps
    a.logits, a.target, a.loss = logits.data_ptr(), t.data_ptr(), out["loss"].data_ptr()
    if with_topk:
        a.correct1, a.correct5 = out["c1"].data_ptr(), out["c5"].data_ptr()
    if with_g:
        a.G, a.ldg = out["G"].data_ptr(), c.ldg
    _run(lib.yamb_softmax_ce_fwd, a)
    for k in ("loss", "c1", "c5"):
        _check_guard(out[k], c.N, "softmax_ce " + k)
    G = out["G"]
    assert bool((G[:, c.C:] == SENTINEL).all()) and bool((G[c.N] == SENTINEL).all()), \
        "softmax_ce G: written outside [N, C)"
    return out


def _ce_loc(n, col=None):
    s = "(row %d: CTA %d, warp %d" % (n, n // 8, n % 8)
    if col is not None:
        s += ", lane %d, step %d" % (col % 32, col // 32)
    return s + ")"


def _check_ce_fwd(lib, c):
    logits, t, _ = _ce_data(c)
    out = _ce_fwd(lib, c, logits, t)
    again = _ce_fwd(lib, c, logits, t)
    for k in ("loss", "c1", "c5", "G"):
        _same(out[k], again[k], "softmax_ce " + k)
    bare = _ce_fwd(lib, c, logits, t, with_g=False, with_topk=False)
    _same(bare["loss"], out["loss"], "softmax_ce loss without G / top-k")
    assert bool((bare["G"] == SENTINEL).all()) and bool((bare["c1"] == SENTINEL).all())

    N, Cc = c.N, c.C
    eps = float(torch.tensor(c.eps, dtype=torch.float32))
    v = logits[:N, :Cc].double()
    ar = torch.arange(N, device=DEV)
    mx = v.max(1).values
    lse = torch.logsumexp(v, 1)
    vt = v[ar, t]
    sv = v.sum(1)
    loss64 = -(1 - eps) * (vt - lse) - (eps / Cc) * (sv - Cc * lse)
    # error bound of the kernel's operations (module docstring)
    x = v - mx[:, None]
    ex = x.exp()
    se = ex.sum(1)
    chain = math.ceil(Cc / 32) + 5
    d_se = ((ex * ((2 + 1.173 * x.abs()) * 2.0 ** -23 + U * x.abs())).sum(1) + Cc * 2.0 ** -126) \
        / se + chain * U
    lnse = se.log()
    e_lse = 1.01 * d_se + 2.0 ** -21.41 + 3 * 2.0 ** -23 * lnse.abs() + U * lse.abs()
    lpt, slp = vt - lse, sv - Cc * lse
    e_lpt = e_lse + U * lpt.abs()
    e_slp = chain * U * v.abs().sum(1) + Cc * e_lse + U * Cc * lse.abs() + U * slp.abs()
    e_loss = (1 - eps) * e_lpt + (eps / Cc) * e_slp + \
        3 * U * ((1 - eps) * lpt.abs() + (eps / Cc) * slp.abs()) + U * loss64.abs()
    r_loss = _worst((out["loss"][:N].double() - loss64).abs(), e_loss,
                    "softmax_ce loss %s" % (tuple(c),), lambda n: _ce_loc(n))
    # top-1 / top-5: the target's position in a stable descending sort
    order = torch.sort(logits[:N, :Cc].float(), dim=1, descending=True, stable=True).indices
    rank = (order == t[:, None]).int().argmax(1)
    _equal(out["c1"][:N], (rank < 1).float(), "softmax_ce correct1 %s" % (tuple(c),),
           lambda n: _ce_loc(n))
    _equal(out["c5"][:N], (rank < 5).float(), "softmax_ce correct5 %s" % (tuple(c),),
           lambda n: _ce_loc(n))
    # G = softmax - smoothed one-hot
    xl = v - lse[:, None]
    p = xl.exp()
    onehot = torch.zeros_like(v)
    onehot[ar, t] = 1.0
    G64 = p - eps / Cc - (1 - eps) * onehot
    e_p = p * ((2 + 1.173 * xl.abs()) * 2.0 ** -23 + U * xl.abs() + 1.01 * e_lse[:, None]) \
        + 2.0 ** -126
    e_G = e_p + U * (eps / Cc) + U * (1 - eps) * onehot + U * (p + eps / Cc) + U * G64.abs()
    _between(out["G"][:N, :Cc], G64, e_G, "softmax_ce G %s" % (tuple(c),), _ce_loc)
    return out, r_loss


@pytest.mark.parametrize("c", tc.CE_CASES, ids=lambda c: "N%d-C%d-ld%d-ldg%d-ldd%d-eps%g" % c)
def test_softmax_ce(built_lib, c):
    out, r_loss = _check_ce_fwd(built_lib, c)
    print("softmax_ce %s: loss err/bound %.3g" % (tuple(c), r_loss))
    if not tc.ce_has_bwd(c):
        return
    nat = _nat()
    N, Cc = c.N, c.C
    G = out["G"]
    g = torch.Generator(device=DEV).manual_seed(N + Cc)
    dloss = torch.randn(N, device=DEV, generator=g)
    db0 = torch.randn(Cc, device=DEV, generator=g)

    def run(with_bias):
        dl = torch.full((N + 1, c.ldd), SENTINEL, device=DEV, dtype=BF)
        db = _guarded(Cc, SENTINEL)
        db[:Cc] = db0
        a = nat.SoftmaxCeGrad()
        a.N, a.C, a.G, a.ldg = N, Cc, G.data_ptr(), c.ldg
        a.dloss, a.dlogits, a.ldd = dloss.data_ptr(), dl.data_ptr(), c.ldd
        a.dbias = db.data_ptr() if with_bias else None
        _run(built_lib.yamb_softmax_ce_bwd, a)
        assert bool((dl[:, Cc:] == SENTINEL).all()) and bool((dl[N] == SENTINEL).all()), \
            "softmax_ce bwd dlogits: written outside [N, C)"
        _check_guard(db, Cc, "softmax_ce bwd dbias")
        return dl, db

    dl, db = run(True)
    dl2, db2 = run(True)
    _same(dl, dl2, "softmax_ce bwd dlogits")
    _same(db, db2, "softmax_ce bwd dbias")
    dl3, db3 = run(False)
    _same(dl3, dl, "softmax_ce bwd dlogits without dbias")
    assert bool((db3[:Cc] == db0).all()), "softmax_ce bwd: dbias written although NULL"
    grid = tc.ce_bwd_grid(N, torch.cuda.get_device_properties(0).multi_processor_count)

    def loc(n, col):
        cp = col // 2
        return "(row %d, column %d: CTA %d, row step %d, thread %d, pair step %d; grid %d)" % (
            n, col, n % grid, n // grid, cp % 256, cp // 256, grid)

    want = (G[:N, :Cc].double() * dloss.double()[:, None]).float().to(BF)
    _equal(dl[:N, :Cc], want, "softmax_ce bwd dlogits %s" % (tuple(c),), loc)
    d64 = dl[:N, :Cc].double()
    r = d64.sum(0)
    q = (d64 * d64).sum(0).sqrt()
    b0 = db0.double()
    rb = _worst((db[:Cc].double() - b0 - r).abs(),
                _long_bound(r, q) + 2.0 ** -23 * (b0.abs() + r.abs()),
                "softmax_ce bwd dbias %s" % (tuple(c),),
                lambda col: "(column %d: %d row slabs of grid %d)" % (col, grid, grid))
    print("softmax_ce bwd %s: dbias err/bound %.3g" % (tuple(c), rb))


# ---- column sum ------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", tc.COLSUM_CASES, ids=lambda c: "M%d-C%d-ld%d" % c)
def test_colsum(built_lib, c):
    g = torch.Generator(device=DEV).manual_seed(c.M * 13 + c.C)
    X = torch.full((c.M + 1, c.ld), POISON, device=DEV, dtype=BF)
    X[:c.M, :c.C] = torch.randn(c.M, c.C, device=DEV, generator=g).to(BF)
    o0 = torch.randn(c.C, device=DEV, generator=g)

    def run():
        out = _guarded(c.C, SENTINEL)
        out[:c.C] = o0
        _nat().check(built_lib.yamb_colsum_bf16(X.data_ptr(), c.M, c.C, c.ld, out.data_ptr(),
                                                _stream()))
        torch.cuda.synchronize()
        _check_guard(out, c.C, "colsum out")
        return out

    out = run()
    _same(out, run(), "colsum out")
    x64 = X[:c.M, :c.C].double()
    r = x64.sum(0)
    q = (x64 * x64).sum(0).sqrt()
    b0 = o0.double()
    gx, gy = tc.colsum_grid(c.M, c.C)
    rc = _worst((out[:c.C].double() - b0 - r).abs(),
                _long_bound(r, q) + 2.0 ** -23 * (b0.abs() + r.abs()),
                "colsum out %s" % (tuple(c),),
                lambda col: "(column %d: column block %d of %d, thread %d, %d row slabs)" % (
                    col, (col // 2) // 256, gx, (col // 2) % 256, gy))
    print("colsum %s: err/bound %.3g" % (tuple(c), rc))


# ---- refused calls write nothing -------------------------------------------------------------------
def test_refused_calls_write_nothing(built_lib):
    nat = _nat()
    lib = built_lib
    d = _stem_data(2, 37, 37)
    w = torch.randn(64 * 27, device=DEV)
    y = torch.full((2 * 19 * 19 * 64 + 8,), SENTINEL, device=DEV, dtype=BF)
    dh = torch.randn(2 * 19 * 19 * 64 + 64, device=DEV).to(BF)
    dw = torch.full((64 * 27 + 8,), SENTINEL, device=DEV)
    sc = torch.ones(64, device=DEV)
    calls = [
        (lib.yamb_stem_conv_fwd, _stem_args(d, 12, w=w, y=y)),
        (lib.yamb_stem_conv_fwd, _stem_args(d, 72, w=w, y=y)),
        (lib.yamb_stem_conv_wgrad, _stem_args(d, 24, dh=dh, dw=dw)),
        (lib.yamb_stem_conv_wgrad, _stem_args(d, 56, dh=dh, dw=dw)),
    ]
    a = _stem_args(d, 32, dh=dh, dw=dw)
    a.dh = dh.data_ptr() + 8
    calls.append((lib.yamb_stem_conv_wgrad, a))
    for act, scale in ((5, sc), (1, None)):
        e = nat.StemConvEval()
        e.conv = _stem_args(d, 32, w=w, y=y)
        e.scale, e.shift, e.act = nat.ptr(scale), sc.data_ptr(), act
        calls.append((lib.yamb_stem_conv_eval_fwd, e))
    logits = torch.zeros(4, 4104, device=DEV, dtype=BF)
    t = torch.zeros(4, device=DEV, dtype=torch.int64)
    outs = [torch.full((4 + 8,), SENTINEL, device=DEV) for _ in range(3)]
    G = torch.full((5, 4104), SENTINEL, device=DEV, dtype=BF)
    for Cc, ld in ((4097, 4104), (1000, 999)):
        a = nat.SoftmaxCe()
        a.N, a.C, a.ld, a.smoothing = 4, Cc, ld, 0.1
        a.logits, a.target = logits.data_ptr(), t.data_ptr()
        a.loss, a.correct1, a.correct5 = (o.data_ptr() for o in outs)
        a.G, a.ldg = G.data_ptr(), 4104
        calls.append((lib.yamb_softmax_ce_fwd, a))
    dl = torch.full((5, 1004), SENTINEL, device=DEV, dtype=BF)
    db = torch.full((1004,), SENTINEL, device=DEV)
    dloss = torch.ones(4, device=DEV)
    for Cc, ldd in ((999, 1004), (1000, 1001)):
        b = nat.SoftmaxCeGrad()
        b.N, b.C, b.G, b.ldg = 4, Cc, G.data_ptr(), 4104
        b.dloss, b.dlogits, b.ldd, b.dbias = dloss.data_ptr(), dl.data_ptr(), ldd, db.data_ptr()
        calls.append((lib.yamb_softmax_ce_bwd, b))
    for fn, args in calls:
        rc = fn(C.byref(args), _stream())
        assert rc == nat.EINVAL, (fn.__name__, rc, lib.yamb_last_error())
    col = torch.full((1000 + 8,), SENTINEL, device=DEV)
    for Cc, ld in ((999, 1000), (1000, 999)):
        rc = lib.yamb_colsum_bf16(logits.data_ptr(), 4, Cc, ld, col.data_ptr(), _stream())
        assert rc == nat.EINVAL, (rc, lib.yamb_last_error())
    torch.cuda.synchronize()
    for name, buf in (("stem y", y), ("stem dw", dw), ("loss", outs[0]), ("correct1", outs[1]),
                      ("correct5", outs[2]), ("G", G), ("dlogits", dl), ("dbias", db),
                      ("colsum", col)):
        assert bool((buf == SENTINEL).all()), "refused call wrote %s" % name
