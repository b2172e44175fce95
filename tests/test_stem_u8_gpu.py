"""GPU: the uint8 stem entry points (yamb_stem_conv_u8_fwd / _wgrad / _eval_fwd), which normalise
uint8 HWC images inside the kernels, and the uint8 input path of the network built on them.

Kernels, for every case of stem_u8_cases.py and both normalisations:
  * bitwise twins: y, eval y and dw equal the bf16 entry points' on xb = bf16(Normalize(ToTensor(u)))
    computed on the host, for the same weights, dh and initial dw;
  * fp64: the same bounds as test_tail_fp64_gpu.py, with X27 the unfold of xb in fp64 (the values
    the kernels stage): y between the bf16 values of y64 -+ 27 u A; eval y exactly
    bf16(act(fp32(scale h + shift))) for no activation, ReLU and ReLU6, else within the band of the
    fp64 activation; dw within _long_bound + the fp32 add onto dw0;
  * two calls give the same bits; guard values keep SENTINEL; a refused call writes nothing.
u carries 0 and 255 in every image (its first row 0, its last row 255) and one more image of 255
after the N the kernel is given.

Network: a TrainStep fed uint8 batches and one fed the host-normalised bf16 batches, from the same
initialisation, are bitwise equal after three steps (CUDA graph from the third): loss, parameters,
running statistics, EMA shadows; then the validation pass (EvalStep calibration and evaluation with
a partial last batch) gives equal metrics and logits.  MobileNetV2 runs the uint8 stem kernels;
width_mult 1.4 (a 48-channel stem) normalises on the device first."""
import copy
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

import stem_u8_cases as uc
from stem_u8_cases import host_normalize
import tail_cases as tc
from _cfg import load_cfgs
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


# ---- kernels ---------------------------------------------------------------------------------------
class _Data:
    """u [N+1, H, W, 3] uint8 (image N all 255), xb [N+1, H, W, 3] bf16 host-normalised (image N
    POISON), X27 fp64 of xb[:N]."""

    def __init__(self, N, H, W, norm):
        g = torch.Generator().manual_seed(N * 1009 + H * 31 + W)
        u = torch.randint(0, 256, (N + 1, H, W, 3), dtype=torch.uint8, generator=g)
        u[:, 0] = 0
        if H > 1:
            u[:, -1] = 255
        u[N] = 255
        self.N, self.H, self.W, self.norm = N, H, W, norm
        self.plan = tc.stem_plan(N, H, W)
        self.u = u.to(DEV)
        self.xb = torch.full((N + 1, H, W, 3), POISON, dtype=BF)
        self.xb[:N] = host_normalize(u[:N], norm)
        self.xb = self.xb.to(DEV)
        cols = F.unfold(self.xb[:N].double().permute(0, 3, 1, 2), 3, padding=1, stride=2)
        self.X27 = cols.transpose(1, 2).reshape(-1, 27).contiguous()
        del cols
        self.gen = torch.Generator(device=DEV).manual_seed(N * 7 + H * 3 + W)


_DATA = {}


def _data(N, H, W, norm):
    key = (N, H, W, norm)
    if key not in _DATA:
        _DATA.clear()
        _DATA[key] = _Data(N, H, W, norm)
    return _DATA[key]


def _u8_args(d, Cout, w=None, y=None, dh=None, dw=None, scale=None, shift=None, act=0):
    nat = _nat()
    a = nat.StemConvU8()
    c = a.ev.conv
    c.N, c.H, c.W, c.Cout = d.N, d.H, d.W, Cout
    c.x = d.u.data_ptr()
    c.w, c.y, c.dh, c.dw = (nat.ptr(t) for t in (w, y, dh, dw))
    a.ev.scale, a.ev.shift, a.ev.act = nat.ptr(scale), nat.ptr(shift), act
    a.mean[:] = d.norm[0]
    a.std[:] = d.norm[1]
    return a


def _bf_args(d, Cout, w=None, y=None, dh=None, dw=None):
    nat = _nat()
    a = nat.StemConv()
    a.N, a.H, a.W, a.Cout = d.N, d.H, d.W, Cout
    a.x = d.xb.data_ptr()
    a.w, a.y, a.dh, a.dw = (nat.ptr(t) for t in (w, y, dh, dw))
    return a


def _bits_equal(a, b, what):
    assert torch.equal(a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8)), \
        "%s: uint8 entry differs from its bf16 twin on the host-normalised image" % what


def _loc(plan):
    def loc(n, oy, ox, *_):
        return "(image %d, tile row %d of %d, tile column %d of %d)" % (
            n, oy // tc.STEM_TH, plan.tiles_h, ox // tc.STEM_TW, plan.tiles_w)
    return loc


def _check_fwd(lib, c, norm):
    d = _data(c.N, c.H, c.W, norm)
    p = d.plan
    n = c.N * p.Ho * p.Wo * c.Cout
    w = torch.randn(c.Cout, 3, 3, 3, device=DEV, generator=d.gen) * 0.3

    def run(fn, args_of):
        buf = _guarded(n, SENTINEL, BF)
        _run(fn, args_of(buf))
        _check_guard(buf, n, "stem u8 fwd y")
        return buf

    buf = run(lib.yamb_stem_conv_u8_fwd, lambda b: _u8_args(d, c.Cout, w=w, y=b))
    _same(buf, run(lib.yamb_stem_conv_u8_fwd, lambda b: _u8_args(d, c.Cout, w=w, y=b)),
          "stem u8 fwd y")
    what = "stem u8 fwd y %s %s" % (tuple(c), norm)
    _bits_equal(buf, run(lib.yamb_stem_conv_fwd, lambda b: _bf_args(d, c.Cout, w=w, y=b)), what)
    W27 = w.double().view(c.Cout, 27)
    y64 = (d.X27 @ W27.t()).view(c.N, p.Ho, p.Wo, c.Cout)
    A = (d.X27.abs() @ W27.abs().t()).view(c.N, p.Ho, p.Wo, c.Cout)
    y = buf[:n].view(c.N, p.Ho, p.Wo, c.Cout)
    _between(y, y64, 27 * U * A, what, _loc(p))
    return w, y


def _check_wgrad(lib, c, norm):
    d = _data(c.N, c.H, c.W, norm)
    p = d.plan
    g = d.gen
    dhbuf = torch.full((c.N + 1, p.Ho, p.Wo, c.Cout), POISON, device=DEV, dtype=BF)
    dhbuf[:c.N] = torch.randn(c.N, p.Ho, p.Wo, c.Cout, device=DEV, generator=g).to(BF)
    n = c.Cout * 27
    dw0 = torch.randn(n, device=DEV, generator=g)

    def run(fn, args_of):
        dw = _guarded(n)
        dw[:n] = dw0
        _run(fn, args_of(dw))
        _check_guard(dw, n, "stem u8 wgrad dw")
        return dw

    dw = run(lib.yamb_stem_conv_u8_wgrad, lambda b: _u8_args(d, c.Cout, dh=dhbuf, dw=b))
    _same(dw, run(lib.yamb_stem_conv_u8_wgrad, lambda b: _u8_args(d, c.Cout, dh=dhbuf, dw=b)),
          "stem u8 wgrad dw")
    what = "stem u8 wgrad dw %s %s" % (tuple(c), norm)
    _bits_equal(dw, run(lib.yamb_stem_conv_wgrad, lambda b: _bf_args(d, c.Cout, dh=dhbuf, dw=b)),
                what)
    dh64 = dhbuf[:c.N].double().view(-1, c.Cout)
    r = dh64.t() @ d.X27
    q = ((dh64 * dh64).t() @ (d.X27 * d.X27)).sqrt()
    b0 = dw0.double().view(c.Cout, 27)
    err = (dw[:n].double().view(c.Cout, 27) - b0 - r).abs()
    return _worst(err, _long_bound(r, q) + 2.0 ** -23 * (b0.abs() + r.abs()), what)


@pytest.mark.parametrize("norm", sorted(uc.NORMS))
@pytest.mark.parametrize("c", uc.DIRECT_CASES, ids=lambda c: "N%d-%dx%d-co%d" % c)
def test_stem_u8_direct(built_lib, c, norm):
    _check_fwd(built_lib, c, uc.NORMS[norm])
    if c.Cout in tc.STEM_WGRAD_COUT:
        _check_wgrad(built_lib, c, uc.NORMS[norm])


@pytest.mark.parametrize("c", uc.WALK_CASES, ids=lambda c: "N%d-%dx%d-co%d" % c)
def test_stem_u8_walk(built_lib, c):
    plan = tc.stem_plan(c.N, c.H, c.W)
    assert tc.stem_is_walk(plan, torch.cuda.get_device_properties(0).multi_processor_count), plan
    _check_fwd(built_lib, c, uc.NORMS["imagenet"])
    r = _check_wgrad(built_lib, c, uc.NORMS["imagenet"])
    print("stem u8 walk %s: wgrad err/bound %.3g" % (tuple(c), r))


@pytest.mark.parametrize("norm", sorted(uc.NORMS))
@pytest.mark.parametrize("cout", tc.STEM_EVAL_COUT)
@pytest.mark.parametrize("shape", uc.EVAL_SHAPES, ids=lambda s: "N%d-%dx%d" % s)
def test_stem_u8_eval(built_lib, shape, cout, norm):
    nat = _nat()
    c = tc.StemCase(*shape, cout)
    w, h = _check_fwd(built_lib, c, uc.NORMS[norm])
    d = _data(*shape, uc.NORMS[norm])
    p = d.plan
    n = c.N * p.Ho * p.Wo * cout
    g = torch.Generator(device=DEV).manual_seed(cout)
    for act in range(5):
        scale = torch.rand(cout, device=DEV, generator=g) + 0.5
        shift = torch.randn(cout, device=DEV, generator=g) * 0.3

        def run_u8():
            buf = _guarded(n, SENTINEL, BF)
            _run(built_lib.yamb_stem_conv_u8_eval_fwd,
                 _u8_args(d, cout, w=w, y=buf, scale=scale, shift=shift, act=act))
            _check_guard(buf, n, "stem u8 eval y")
            return buf

        buf = run_u8()
        _same(buf, run_u8(), "stem u8 eval y")
        twin = _guarded(n, SENTINEL, BF)
        e = nat.StemConvEval()
        e.conv = _bf_args(d, cout, w=w, y=twin)
        e.scale, e.shift, e.act = scale.data_ptr(), shift.data_ptr(), act
        _run(built_lib.yamb_stem_conv_eval_fwd, e)
        what = "stem u8 eval y %s act %d %s" % (tuple(c), act, norm)
        _bits_equal(buf, twin, what)
        y = buf[:n].view_as(h)
        z32 = _f32(h.double() * scale.double() + shift.double())
        if act in (0, 1, 2):
            _equal(y, _clamp32(z32, act).to(BF), what, _loc(p))
        else:
            a64 = _act64(z32, act)
            _between(y, a64, (BAND + 2.0 ** -22) * a64.abs(), what, _loc(p))


def test_stem_u8_refused_calls_write_nothing(built_lib):
    lib = built_lib
    d = _data(2, 36, 44, uc.NORMS["imagenet"])
    w = torch.randn(64 * 27, device=DEV)
    y = torch.full((2 * 18 * 22 * 64 + 16,), SENTINEL, device=DEV, dtype=BF)
    dh = torch.randn(2 * 18 * 22 * 64 + 64, device=DEV).to(BF)
    dw = torch.full((64 * 27 + 8,), SENTINEL, device=DEV)
    sc = torch.ones(64, device=DEV)
    entries = [(lib.yamb_stem_conv_u8_fwd, dict(w=w, y=y)),
               (lib.yamb_stem_conv_u8_eval_fwd, dict(w=w, y=y, scale=sc, shift=sc, act=1)),
               (lib.yamb_stem_conv_u8_wgrad, dict(dh=dh, dw=dw))]
    calls = []
    for fn, kw in entries:
        for cout in (12, 72):
            calls.append((fn, _u8_args(d, cout, **kw)))
        for bad in (0.0, float("nan"), float("inf")):
            a = _u8_args(d, 32, **kw)
            a.std[1] = bad
            calls.append((fn, a))
        a = _u8_args(d, 32, **kw)
        a.mean[2] = float("nan")
        calls.append((fn, a))
        a = _u8_args(d, 32, **kw)
        a.ev.conv.x = None
        calls.append((fn, a))
    calls.append((lib.yamb_stem_conv_u8_wgrad, _u8_args(d, 24, dh=dh, dw=dw)))
    for fn, kw in entries[:2]:
        a = _u8_args(d, 32, **kw)
        a.ev.conv.y = y.data_ptr() + 8
        calls.append((fn, a))
    for fn, args in calls:
        rc = fn(C.byref(args), _stream())
        assert rc == _nat().EINVAL, (fn.__name__, rc, lib.yamb_last_error())
    torch.cuda.synchronize()
    for name, buf in (("stem u8 y", y), ("stem u8 dw", dw)):
        assert bool((buf == SENTINEL).all()), "refused call wrote %s" % name


@pytest.mark.parametrize("norm", sorted(uc.NORMS))
def test_device_normalize_matches_host(built_lib, norm):
    """The fallback of a stem the kernels do not cover: every byte value in every channel."""
    from yet_another_mobilenet_series_b200 import tail_ops
    u = torch.arange(256, dtype=torch.uint8).repeat(3, 1).t().reshape(1, 16, 16, 3)
    u = torch.cat([u, u.flip(1)])
    got = tail_ops.normalize_u8(u.to(DEV).permute(0, 3, 1, 2), uc.NORMS[norm])
    want = host_normalize(u, uc.NORMS[norm]).permute(0, 3, 1, 2)
    assert got.is_contiguous(memory_format=torch.channels_last)
    _bits_equal(got.cpu(), want.contiguous(), "normalize_u8 %s" % norm)


# ---- network ---------------------------------------------------------------------------------------
SIZE, B = 96, 8


def _model(width_mult):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    from yet_another_mobilenet_series_b200 import mobilenet_supernet as sup
    kw = dict(load_cfgs()["mobilenet_v2"]["model_kwparams"])
    kw.update(width_mult=width_mult, num_classes=100, input_size=SIZE, dropout_ratio=0.0)
    torch.manual_seed(5)
    m = sup.Model(**kw)
    m.apply(mb.init_weights_mnas)
    return m


def _batches(g, n, norm, count, last=None):
    out = []
    for i in range(count):
        bn = last if (last is not None and i == count - 1) else n
        u = torch.randint(0, 256, (bn, SIZE, SIZE, 3), dtype=torch.uint8, generator=g)
        u[:, 0] = 0
        u[:, -1] = 255
        t = torch.randint(0, 100, (bn,), generator=g)
        xu = u.permute(0, 3, 1, 2)                                  # NCHW, channels_last storage
        xb = host_normalize(u, norm).permute(0, 3, 1, 2)
        out.append(((xu, t), (xb, t)))
    return out


@pytest.mark.parametrize("width_mult", (1.0, 1.4))
def test_uint8_train_and_eval_match_host_normalised(built_lib, width_mult):
    from yet_another_mobilenet_series_b200 import engine, tail_ops
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    norm = uc.NORMS["imagenet"]
    dev = torch.device("cuda")
    m_u8 = _model(width_mult)
    m_bf = copy.deepcopy(m_u8)
    stem = m_u8.features[0]
    covered = tail_ops.stem_supported(stem, torch.empty(1, device=dev))
    assert covered == (width_mult == 1.0), stem
    m_u8, m_bf = m_u8.to(dev), m_bf.to(dev)
    ts_u8 = TrainStep(m_u8, B, image_size=SIZE, input_dtype=torch.uint8, input_norm=norm)
    ts_bf = TrainStep(m_bf, B, image_size=SIZE)
    assert ts_u8.x.dtype == torch.uint8 and ts_u8.x.is_contiguous(memory_format=torch.channels_last)
    g = torch.Generator().manual_seed(11)
    for (xu, t), (xb, _) in _batches(g, B, norm, 3):
        lu, lb = ts_u8(xu, t), ts_bf(xb, t)
        torch.cuda.synchronize()
        _bits_equal(lu, lb, "loss")
    assert ts_u8.graph is not None and ts_bf.graph is not None
    for (k, a), b in zip(m_u8.named_parameters(), m_bf.parameters()):
        _bits_equal(a.detach(), b.detach(), "parameter " + k)
        _bits_equal(ts_u8.opt.ema_shadow(a), ts_bf.opt.ema_shadow(b), "EMA of " + k)
    for (k, a), b in zip(m_u8.named_buffers(), m_bf.buffers()):
        _bits_equal(a, b, "buffer " + k)
    for a, b in zip(ts_u8.stat_shadow, ts_bf.stat_shadow):
        _bits_equal(a, b, "EMA of a running statistic")
    # validation: calibration on 2 full batches, evaluation on 2 full + 1 partial batch
    calib = _batches(g, B, norm, 2)
    val = _batches(g, B, norm, 3, last=5)
    n0 = engine.EVAL_TAIL_CALLS
    r_u8 = ts_u8.validate([a for a, _ in val], calib_batches=[a for a, _ in calib])
    r_bf = ts_bf.validate([b for _, b in val], calib_batches=[b for _, b in calib])
    assert engine.EVAL_TAIL_CALLS > n0
    assert r_u8 == r_bf, (r_u8, r_bf)
    assert ts_u8._eval_step.logits.shape[0] == 5
    _bits_equal(ts_u8._eval_step.logits, ts_bf._eval_step.logits, "logits of the partial batch")
    ema_u8, ema_bf = ts_u8.ema_model(), ts_bf.ema_model()
    assert ema_u8.input_norm == (tuple(norm[0]), tuple(norm[1]))
    with torch.no_grad():
        xu, xb = val[0][0][0], val[0][1][0]
        _bits_equal(ema_u8(xu.to(dev)), ema_bf(xb.to(dev)), "eval forward of a full batch")


def test_uint8_without_norm_unchanged(built_lib):
    """A model without an input normalisation takes a uint8 batch as it always did: its values
    0..255 cast to bf16."""
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    m = _model(1.0).to("cuda").eval()
    with pytest.raises(ValueError):
        TrainStep(m, B, image_size=SIZE, input_dtype=torch.uint8)
    g = torch.Generator().manual_seed(3)
    u = torch.randint(0, 256, (4, SIZE, SIZE, 3), dtype=torch.uint8, generator=g)
    xu = u.permute(0, 3, 1, 2).to("cuda")
    with torch.no_grad():
        _bits_equal(m(xu), m(xu.to(BF)), "uint8 input without a norm")


def test_prefetcher_hands_over_uint8_batches_byte_for_byte():
    import numpy as np
    from yet_another_mobilenet_series_b200.dataflow import DataPrefetcher, fast_collate
    rng = np.random.default_rng(4)
    loader = [fast_collate([(rng.integers(0, 256, (20, 28, 3), dtype=np.uint8), int(k))
                            for k in rng.integers(0, 1000, n)]) for n in (4, 4, 3)]
    got = [(x.cpu(), t.cpu(), x.is_contiguous(memory_format=torch.channels_last))
           for x, t in DataPrefetcher(loader, dtype=torch.uint8)]
    assert len(got) == len(loader)
    for (x, t, cl), (xs, ts) in zip(got, loader):
        assert cl and x.dtype == torch.uint8 and x.shape == xs.shape
        assert torch.equal(x, xs) and torch.equal(t, ts)
