"""GPU: the training-mode Squeeze-and-Excitation backward (TrainStep(fused_se=True)).

- yamb_se_bwd_stats_bwd: dgate bitwise that of yamb_se_bwd_reduce_bwd; A, B, A', B' against fp64
  sums of the same bf16 inputs, element by element, within gam(L)*sum|terms| for the fp32
  per-thread chains (L bounded by the pixels of a sample, plus the act' and xhat roundings).
- yamb_se_bn_bwd_finalize: ca, cb, cc, dgamma, dbeta against an fp64 BatchNorm backward of the
  fp64 dz2 sums, element by element.
- yamb_depthwise_bwd_se, every (k, stride, channel tile) with and without the expansion, on
  multi-tile walks, odd maps and stride 2: dx (or dz1 and the BatchNorm-1 backward) and dw bitwise
  those of yamb_se_bwd_apply_bwd followed by yamb_depthwise_bwd with the same ca / cb / cc.
- Three TrainStep(fused_se=True) steps of atomnas_c+ and autonl_l against the fp32 reference step
  under the autocast yardstick, also with fused_stem + fused_tail; with micro_batch against the
  default step with the same micro_batch.
- Two runs and eager / graph replay give the same bits; a network without SE gives the default's
  bits."""
import ctypes as C
import sys
import types

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture
def flags(monkeypatch):
    mod = types.ModuleType("utils.config")
    mod.FLAGS = types.SimpleNamespace()
    monkeypatch.setitem(sys.modules, "utils.config", mod)
    return mod


def _bf(*shape, g, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).cuda()


def _f(*shape, g, lo=-1.0, hi=1.0):
    return (torch.rand(*shape, generator=g) * (hi - lo) + lo).cuda()


def _call(fn, a):
    from yet_another_mobilenet_series_b200 import native as nat
    nat.check(fn(C.byref(a), nat.stream_handle()))


def _actd(z, act):
    """act'(z) in fp64 of fp32 z (ReLU6 / Swish)."""
    z = z.double()
    if act == 2:
        return ((z > 0) & (z < 6)).double()
    s = torch.sigmoid(z)
    return s * (1 + z * (1 - s))


# ---- se_bwd_stats -------------------------------------------------------------------------------
@pytest.mark.parametrize("N,HW,C,act", [(4, 196, 144, 2), (3, 49, 40, 3), (2, 784, 16, 2),
                                        (2, 49, 2304, 3)])
def test_stats_vs_reduce_and_fp64(built_lib, N, HW, C, act):
    from yet_another_mobilenet_series_b200 import native as nat
    g = torch.Generator().manual_seed(N * HW + C)
    dy, h = _bf(N * HW, C, g=g), _bf(N * HW, C, g=g)
    sc, sh = _f(C, g=g, lo=0.5, hi=1.5), _f(C, g=g, lo=-0.5, hi=0.5)
    mu, rs = _f(C, g=g, lo=-0.2, hi=0.2), _f(C, g=g, lo=0.5, hi=2.0)
    dg0 = torch.zeros(N, C, device="cuda")
    r = nat.SeBwdReduce()
    r.N, r.HW, r.C, r.ldd, r.ldh = N, HW, C, C, C
    r.dy, r.h, r.scale, r.shift, r.act = dy.data_ptr(), h.data_ptr(), sc.data_ptr(), sh.data_ptr(), act
    r.dgate = dg0.data_ptr()
    _call(built_lib.yamb_se_bwd_reduce_bwd, r)
    outs = []
    for _ in range(2):
        dg = torch.full((N, C), float("nan"), device="cuda")
        sums = torch.full((4, N, C), float("nan"), device="cuda", dtype=torch.float64)
        s = nat.SeBwdStats()
        s.N, s.HW, s.C, s.ldd, s.ldh = N, HW, C, C, C
        s.dy, s.h, s.scale, s.shift, s.act = dy.data_ptr(), h.data_ptr(), sc.data_ptr(), \
            sh.data_ptr(), act
        s.mean, s.invstd, s.dgate, s.sums = mu.data_ptr(), rs.data_ptr(), dg.data_ptr(), \
            sums.data_ptr()
        _call(built_lib.yamb_se_bwd_stats_bwd, s)
        outs.append((dg, sums))
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], dg0), "dgate differs from se_bwd_reduce"
    assert torch.equal(outs[0][1], outs[1][1]), "sums differ run to run"
    sums = outs[0][1]
    d64, h64 = dy.double().view(N, HW, C), h.double().view(N, HW, C)
    z32 = (sc.double() * h64 + sh.double()).float()
    ad = _actd(z32, act)
    xh = (h64 - mu.double()) * rs.double()
    terms = [d64 * ad, ad, d64 * ad * xh, ad * xh]
    gam = (HW + 12) * 2.0 ** -24
    for k, t in enumerate(terms):
        ref, mag = t.sum(1), t.abs().sum(1)
        err = (sums[k] - ref).abs()
        bound = gam * mag * 1.01 + 1e-30
        worst = float((err / bound).max())
        assert worst <= 1.0, "sum %d: err/bound %.3f" % (k, worst)


# ---- se_bn_bwd_finalize --------------------------------------------------------------------------
@pytest.mark.parametrize("N,Cc,c0,Chid", [(32, 144, 0, 144), (5, 24, 16, 56), (256, 40, 0, 40)])
def test_finalize_vs_fp64(built_lib, N, Cc, c0, Chid):
    from yet_another_mobilenet_series_b200 import native as nat
    g = torch.Generator().manual_seed(N + Cc)
    count = N * 49
    sums = (torch.randn(4, N, Chid, generator=g, dtype=torch.float64) * 10).cuda()
    gate, dpool = _f(N, Chid, g=g, lo=0, hi=1), _f(N, Chid, g=g, lo=-0.1, hi=0.1)
    gamma, mu, rs = _f(Cc, g=g, lo=0.5, hi=1.5), _f(Cc, g=g, lo=-0.5, hi=0.5), _f(Cc, g=g, lo=0.5, hi=2)
    dgam, dbet = _f(Cc, g=g), _f(Cc, g=g)
    dgam0, dbet0 = dgam.clone(), dbet.clone()
    ca, cb, cc = (torch.full((Cc,), float("nan"), device="cuda") for _ in range(3))
    bn = nat.BnBwd()
    bn.gamma, bn.mean, bn.invstd = gamma.data_ptr(), mu.data_ptr(), rs.data_ptr()
    bn.dgamma, bn.dbeta = dgam.data_ptr(), dbet.data_ptr()
    bn.ca, bn.cb, bn.cc = ca.data_ptr(), cb.data_ptr(), cc.data_ptr()
    bn.count, bn.use_batch_stats = count, 1
    f = nat.SeBnBwdFinalize()
    f.N, f.C, f.lds, f.ldg = N, Cc, Chid, Chid
    f.sums, f.gate, f.dpool = sums.data_ptr() + 8 * c0, gate.data_ptr() + 4 * c0, \
        dpool.data_ptr() + 4 * c0
    f.bn = C.pointer(bn)
    _call(built_lib.yamb_se_bn_bwd_finalize, f)
    torch.cuda.synchronize()
    s_ = slice(c0, c0 + Cc)
    G, P = gate[:, s_].double(), dpool[:, s_].double()
    s = (G * sums[0][:, s_] + P * sums[1][:, s_]).sum(0)
    q = (G * sums[2][:, s_] + P * sums[3][:, s_]).sum(0)
    u = 2.0 ** -24
    assert ((dbet.double() - (dbet0.double() + s)).abs() <= 2 * u * (dbet0.double().abs() + s.abs()) + 1e-30).all()
    assert ((dgam.double() - (dgam0.double() + q)).abs() <= 2 * u * (dgam0.double().abs() + q.abs()) + 1e-30).all()
    scd = gamma.double() * rs.double()
    m1, m2 = s / count, q / count
    assert ((ca.double() - scd).abs() <= u * scd.abs()).all()
    cb_ref = -scd * rs.double() * m2
    assert ((cb.double() - cb_ref).abs() <= 6 * u * cb_ref.abs() + 1e-30).all()
    t1, t2 = mu.double() * rs.double() * m2, m1
    cc_ref = scd * (t1 - t2)
    assert ((cc.double() - cc_ref).abs() <= 8 * u * scd.abs() * (t1.abs() + t2.abs()) + 1e-30).all()


# ---- depthwise_bwd_se against se_bwd_apply + depthwise_bwd ---------------------------------------
# (k, stride, C, H, W, expand): C and H pick the channel tile (8: C <= 8, H >= 28; 16: C <= 16,
# H >= 14; 32: C <= 32 or C = 96; 64 otherwise); odd maps, multi-tile walks, stride 2
DW_CASES = [(k, s, c, h, w, e) for k in (3, 5, 7) for s in (1, 2)
            for (c, h, w) in ((8, 37, 29), (16, 29, 17), (32, 15, 19), (96, 14, 14), (128, 9, 13))
            for e in (True, False) if not (not e and c == 96)]


def _dw_case(k, s, Cc, H, W, expand, g):
    N, Chid, c0 = 2, Cc + 16, 8
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    t = {"dy": _bf(N * Ho * Wo, Chid, g=g), "h": _bf(N * Ho * Wo, Chid, g=g),
         "x": _bf(N * H * W, Chid, g=g), "res": _bf(N * H * W, Chid, g=g),
         "gate": _f(N, Chid, g=g, lo=0, hi=1), "dpool": _f(N, Chid, g=g, lo=-0.2, hi=0.2),
         "sc2": _f(Chid, g=g, lo=0.5, hi=1.5), "sh2": _f(Chid, g=g, lo=-0.5, hi=0.5),
         "ca": _f(Chid, g=g), "cb": _f(Chid, g=g, lo=-0.1, hi=0.1), "cc": _f(Chid, g=g, lo=-0.1, hi=0.1),
         "w": _f(Chid, k * k, g=g), "sc1": _f(Chid, g=g, lo=0.5, hi=1.5),
         "sh1": _f(Chid, g=g, lo=-0.5, hi=0.5), "mu1": _f(Chid, g=g, lo=-0.2, hi=0.2),
         "rs1": _f(Chid, g=g, lo=0.5, hi=2.0), "gam1": _f(Chid, g=g, lo=0.5, hi=1.5)}
    return N, Chid, c0, Ho, Wo, t


def _dw_struct(nat, N, H, W, Cc, Chid, c0, k, s, dz, t, dw, dx, bn1, expand, act1):
    d = nat.DwBwd()
    d.N, d.H, d.W, d.C, d.ldc, d.k, d.stride = N, H, W, Cc, Chid, k, s
    d.dz, d.h = dz.data_ptr() + 2 * c0, t["h"].data_ptr() + 2 * c0
    d.ca, d.cb, d.cc = (t[n].data_ptr() + 4 * c0 for n in ("ca", "cb", "cc"))
    d.w, d.dw = t["w"].data_ptr() + 4 * c0 * k * k, dw.data_ptr()
    d.x, d.dx = t["x"].data_ptr() + 2 * c0, dx.data_ptr() + 2 * c0
    d.in_scale, d.in_shift, d.in_act = t["sc1"].data_ptr() + 4 * c0, t["sh1"].data_ptr() + 4 * c0, act1
    if not expand:
        d.residual = t["res"].data_ptr() + 2 * c0
    d.bn = C.pointer(bn1)
    return d


def _act64(z, act):
    """act(z) and act'(z) in fp64 of fp32 z (csrc/prims.cuh act_fwd / act_bwd)."""
    z = z.double()
    if act == 2:
        return z.clamp(0, 6), ((z > 0) & (z < 6)).double()
    if act == 3:
        sg = torch.sigmoid(z)
        return z * sg, sg * (1 + z * (1 - sg))
    r = (z + 3).clamp(0, 6)
    d = torch.where(z <= -3, torch.zeros_like(z), torch.where(z >= 3, torch.ones_like(z), (2 * z + 3) / 6))
    return z * r / 6, d


def _fp32_fma(a, b, c):
    """fp32 fmaf(a, b, c) of fp32 / bf16 operands: the product is exact in fp64."""
    return (a.double() * b.double() + c.double()).float()


def _nchw(m, N, H, W, c0, Cc):
    return m.view(N, H, W, -1)[..., c0:c0 + Cc].permute(0, 3, 1, 2).double()


def _dw_fp64(t, N, H, W, Ho, Wo, Cc, c0, k, s, expand, act1, act2):
    """fp64 dx [N, Cc, H, W] and dw [Cc, k*k] of the SE depthwise backward and their bounds.  Every bf16
    rounding the kernels make (dz2, dh, a1, dx) is allowed half a bf16 ulp (2^-8 relative) and
    every fp32 expression a few fp32 ulps (64 u for the fast-math exp of Swish); the fp32 sums
    gam(n) * sum|terms| with n the taps (dx) or the pixels (dw)."""
    u, b = 2.0 ** -24, 2.0 ** -8
    sl = slice(c0, c0 + Cc)
    dy, h = _nchw(t["dy"], N, Ho, Wo, c0, Cc), _nchw(t["h"], N, Ho, Wo, c0, Cc)
    per = lambda v: v[sl].double().view(1, -1, 1, 1)
    gate = t["gate"][:, sl].double().view(N, Cc, 1, 1)
    dpool = t["dpool"][:, sl].double().view(N, Cc, 1, 1)
    z2 = _fp32_fma(per(t["sc2"]), h, per(t["sh2"])).double()
    _, d2 = _act64(z2, act2)
    pre = dy * gate + dpool
    dz = pre * d2
    e_dz = b * dz.abs() + 64 * u * pre.abs() * (d2.abs() + 1)
    ca, cb, cc = per(t["ca"]), per(t["cb"]), per(t["cc"])
    dh = ca * dz + cb * h + cc
    e_dh = ca.abs() * e_dz * (1 + b) + b * dh.abs() + 4 * u * ((ca * dz).abs() + (cb * h).abs() + cc.abs())
    x = _nchw(t["x"], N, H, W, c0, Cc)
    z1 = _fp32_fma(per(t["sc1"]), x, per(t["sh1"])).double()
    a1, d1 = _act64(z1, act1)
    e_a1 = (b + 64 * u) * a1.abs()
    w = t["w"][sl].double().view(Cc, 1, k, k)
    pad = (k - 1) // 2

    def conv_grads(inp, wt, up):
        inp, wt = inp.clone().requires_grad_(True), wt.clone().requires_grad_(True)
        torch.nn.functional.conv2d(inp, wt, stride=s, padding=pad, groups=Cc).backward(up)
        return inp.grad, wt.grad.view(Cc, k * k)

    da, dw = conv_grads(a1, w, dh)
    s_da, s_dw = conv_grads(a1.abs(), w.abs(), dh.abs())
    e_da = conv_grads(a1.abs(), w.abs(), e_dh)[0] + (k * k + 2) * u * s_da
    e_dw = conv_grads(a1.abs(), w.abs(), e_dh)[1] + conv_grads(e_a1, w.abs(), dh.abs())[1] + \
        (N * Ho * Wo + 2) * u * s_dw
    dx = da * d1
    e_dx = d1.abs() * e_da + 64 * u * da.abs()
    if not expand:
        dx = dx + _nchw(t["res"], N, H, W, c0, Cc)
    return dx, e_dx + b * dx.abs() + 1e-30, dw, e_dw + 1e-30


def _dw_fp64_check(got, t, N, H, W, Ho, Wo, Cc, c0, k, s, expand, act1, act2):
    """dw and dx of the SE depthwise backward against fp64, element by element (_dw_fp64)."""
    dx, e_dx, dw, e_dw = _dw_fp64(t, N, H, W, Ho, Wo, Cc, c0, k, s, expand, act1, act2)
    got_dx = _nchw(got["dx"], N, H, W, c0, Cc)
    rx = float(((got_dx - dx).abs() / e_dx).max())
    rw = float(((got["dw"].double() - dw).abs() / e_dw).max())
    assert rx <= 1.0 and rw <= 1.0, "err/bound dx %.3f dw %.3f" % (rx, rw)


# BatchNorm-2 activation (the SE path's act') and a different BatchNorm-1 activation
ACTS = [(2, 3), (3, 4), (4, 2)]


@pytest.mark.parametrize("act2,act1", ACTS)
@pytest.mark.parametrize("k,s,Cc,H,W,expand", DW_CASES)
def test_depthwise_bwd_se_bitwise(built_lib, k, s, Cc, H, W, expand, act2, act1):
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200 import native as nat
    g = torch.Generator().manual_seed(k * 1000 + s * 100 + Cc + H)
    N, Chid, c0, Ho, Wo, t = _dw_case(k, s, Cc, H, W, expand, g)
    ws = engine.Workspace.get(torch.device("cuda"))
    res = []
    for fused in (False, True, True):
        dw = torch.zeros(Cc, k * k, device="cuda")
        dx = torch.zeros(N * H * W, Chid, device="cuda", dtype=torch.bfloat16)
        o1 = {n: torch.full((Cc,), float("nan"), device="cuda") for n in ("ca", "cb", "cc")}
        dg1, db1 = torch.zeros(Cc, device="cuda"), torch.zeros(Cc, device="cuda")
        bn1 = nat.BnBwd()
        bn1.partials, bn1.counter = ws.stats(Cc)
        bn1.gamma, bn1.mean, bn1.invstd = (t[n].data_ptr() + 4 * c0 for n in ("gam1", "mu1", "rs1"))
        bn1.dgamma, bn1.dbeta = dg1.data_ptr(), db1.data_ptr()
        bn1.ca, bn1.cb, bn1.cc = (o1[n].data_ptr() for n in ("ca", "cb", "cc"))
        bn1.count, bn1.use_batch_stats = N * H * W, 1
        if not fused:
            dz = t["dy"].clone()
            bn2 = nat.BnBwd()       # se_bwd_apply's own BN-2 finalize goes to scratch outputs
            bn2.partials, bn2.counter = ws.stats(Cc)
            scratch = [torch.zeros(Cc, device="cuda") for _ in range(5)]
            bn2.mean, bn2.invstd = t["mu1"].data_ptr() + 4 * c0, t["rs1"].data_ptr() + 4 * c0
            bn2.ca, bn2.cb, bn2.cc = (x.data_ptr() for x in scratch[:3])
            bn2.dgamma, bn2.dbeta = scratch[3].data_ptr(), scratch[4].data_ptr()
            bn2.count, bn2.use_batch_stats = N * Ho * Wo, 1
            a = nat.SeBwdApply()
            a.M, a.C, a.ldd, a.ldh, a.ldz, a.rows_per_sample = N * Ho * Wo, Cc, Chid, Chid, Chid, Ho * Wo
            a.dy = a.dz = dz.data_ptr() + 2 * c0
            a.h = t["h"].data_ptr() + 2 * c0
            a.scale, a.shift, a.act = t["sc2"].data_ptr() + 4 * c0, t["sh2"].data_ptr() + 4 * c0, act2
            a.gate, a.dpool, a.ldg = t["gate"].data_ptr() + 4 * c0, t["dpool"].data_ptr() + 4 * c0, Chid
            a.bn = C.pointer(bn2)
            _call(built_lib.yamb_se_bwd_apply_bwd, a)
            d = _dw_struct(nat, N, H, W, Cc, Chid, c0, k, s, dz, t, dw, dx, bn1, expand, act1)
            _call(built_lib.yamb_depthwise_bwd, d)
        else:
            e = nat.DwBwdSe()
            e.dw = _dw_struct(nat, N, H, W, Cc, Chid, c0, k, s, t["dy"], t, dw, dx, bn1, expand, act1)
            e.gate, e.dpool, e.ldg = t["gate"].data_ptr() + 4 * c0, t["dpool"].data_ptr() + 4 * c0, Chid
            e.scale, e.shift, e.act = t["sc2"].data_ptr() + 4 * c0, t["sh2"].data_ptr() + 4 * c0, act2
            _call(built_lib.yamb_depthwise_bwd_se, e)
        torch.cuda.synchronize()
        res.append({"dw": dw, "dx": dx, "dg1": dg1, "db1": db1, **o1})
    for r in res[1:]:
        for n in res[0]:
            assert torch.equal(res[0][n], r[n]), n
    assert torch.isfinite(res[0]["dw"]).all() and res[0]["dw"].abs().sum() > 0
    _dw_fp64_check(res[1], t, N, H, W, Ho, Wo, Cc, c0, k, s, expand, act1, act2)


# ---- TrainStep(fused_se=True) --------------------------------------------------------------------
def _rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def _flat(d, keys):
    return torch.cat([d[k].detach().double().flatten().cpu() for k in keys])


@pytest.mark.parametrize("name,kw2", [("atomnas_c+", {}), ("autonl_l", {}),
                                      ("atomnas_c+", {"fused_stem": True, "fused_tail": True})])
def test_three_fused_se_steps_vs_fp32_reference(built_lib, flags, name, kw2):
    from _cfg import build_from_cfg
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    B, dev = 16, torch.device("cuda")
    model, cfg = build_from_cfg(name)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    fl = cfg["flags"]
    kw = dict(base_lr=fl["base_lr"], base_total_batch=fl["base_total_batch"], alpha=fl["alpha"],
              momentum=fl["momentum"], eps=fl["epsilon"], weight_decay=fl["weight_decay"],
              label_smoothing=fl["label_smoothing"], ema_decay=fl["moving_average_decay"],
              ema_base_batch=fl["moving_average_decay_base_batch"])
    ref32 = tm.RefTrainer(tm.as_reference(model).to(dev), B, **kw)
    ref16 = tm.RefTrainer(tm.as_reference(model).to(dev).to(memory_format=torch.channels_last), B,
                          autocast=torch.bfloat16, **kw)
    p0 = {k: v.detach().clone() for k, v in model.named_parameters()}
    model = model.to(dev)
    hw = fl["image_size"]
    ts = TrainStep(model, B, image_size=hw, fused_se=True, **kw, **kw2)
    g = torch.Generator().manual_seed(0)
    keys = [k for k, _ in model.named_parameters()]
    n0 = engine.TRAIN_SE_CALLS
    rows = []
    for i in range(3):
        x = torch.randn(B, 3, hw, hw, generator=g).bfloat16()
        t = torch.randint(0, 1000, (B,), generator=g)
        xd, td = x.to(dev).float(), t.to(dev)
        lt = ref32.step(xd, td) - float(tm.l2_loss_mnas(ref32.model, fl["weight_decay"]))
        la = ref16.step(xd.contiguous(memory_format=torch.channels_last), td) - float(
            tm.l2_loss_mnas(ref16.model, fl["weight_decay"]))
        lo = float(ts(x, t))
        rows.append("step %d loss ours %.6f fp32 %.6f autocast %.6f" % (i, lo, lt, la))
        assert abs(lo - lt) <= 2.0 * abs(la - lt) + 5e-3 * abs(lt), rows
    torch.cuda.synchronize()
    assert engine.TRAIN_SE_CALLS > n0 and not engine.TRAIN_SE_FUSED
    pt, pa, po = (dict(m.named_parameters()) for m in (ref32.model, ref16.model, model))
    p0f = _flat(p0, keys)
    eo, ea = _rel(_flat(po, keys) - p0f, _flat(pt, keys) - p0f), _rel(_flat(pa, keys) - p0f,
                                                                     _flat(pt, keys) - p0f)
    rows.append("update rel-L2 ours %.4f autocast %.4f" % (eo, ea))
    assert eo <= 1.3 * ea + 1e-2, rows
    bt, ba, bo = (dict(m.named_buffers()) for m in (ref32.model, ref16.model, model))
    for kind in ("running_mean", "running_var"):
        ks = [k for k in bt if k.endswith(kind)]
        e_o = sorted(_rel(bo[k].cpu(), bt[k].cpu()) for k in ks)
        e_a = sorted(_rel(ba[k].cpu(), bt[k].cpu()) for k in ks)
        mo, ma = sum(e_o) / len(e_o), sum(e_a) / len(e_a)
        qo, qa = e_o[int(0.9 * (len(e_o) - 1))], e_a[int(0.9 * (len(e_a) - 1))]
        rows.append("%s mean ours %.2e autocast %.2e p90 ours %.2e autocast %.2e"
                    % (kind, mo, ma, qo, qa))
        assert mo <= 1.5 * ma + 2e-3 and qo <= 1.5 * qa + 2e-3, rows


def _snap(ts, loss):
    out = {"loss": loss.clone()}
    for n, p in ts.model.named_parameters():
        out["p." + n] = p.detach().clone()
    for n, b in ts.model.named_buffers():
        out["buf." + n] = b.clone()
    return out


def _same(a, b):
    assert a.keys() == b.keys()
    diff = [k for k in a if not torch.equal(a[k], b[k])]
    assert not diff, diff[:5]


def _runs(name, steps=3, B=8, **kw):
    from _cfg import build_from_cfg
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    model, cfg = build_from_cfg(name)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    hw = cfg["flags"]["image_size"]
    ts = TrainStep(model.cuda(), B, image_size=hw, **kw)
    g = torch.Generator().manual_seed(7)
    out = []
    for _ in range(steps):
        x = torch.randn(B, 3, hw, hw, generator=g).bfloat16()
        t = torch.randint(0, 1000, (B,), generator=g)
        out.append(_snap(ts, ts(x, t)))
    return out


def test_micro_batch_close_to_default(built_lib, flags):
    """With micro_batch the fp32 reference step (whole-batch BatchNorm statistics) is not the
    yardstick; the default step with the same micro_batch is: the losses agree to 1e-3 relative,
    and after three RMSprop steps the updates differ by less than the autocast step's update
    differs from the fp32 step's at this size (0.21 rel-L2, test_three_fused_se_steps_vs_fp32_reference;
    measured here on an H100: 0.10)."""
    from _cfg import build_from_cfg
    p0 = {k: v.detach().clone().cuda() for k, v in build_from_cfg("autonl_l")[0].named_parameters()}
    a = _runs("autonl_l", B=16, micro_batch=8, use_graph=False)
    b = _runs("autonl_l", B=16, micro_batch=8, use_graph=False, fused_se=True)
    for x, y in zip(a, b):
        assert abs(float(x["loss"]) - float(y["loss"])) <= 1e-3 * abs(float(x["loss"]))
    keys = ["p." + k for k in p0]
    d0 = torch.cat([(a[-1][k] - p0[k[2:]]).double().flatten() for k in keys])
    d1 = torch.cat([(b[-1][k] - p0[k[2:]]).double().flatten() for k in keys])
    assert float((d1 - d0).norm() / d0.norm()) <= 0.2


def test_graph_replay_equals_eager_and_runs_repeat(built_lib, flags):
    runs = [_runs("atomnas_c+", fused_se=True, use_graph=ug) for ug in (False, True, True)]
    for a, b, c in zip(*runs):
        _same(a, b)
        _same(b, c)


def test_network_without_se_keeps_default_bits(built_lib, flags):
    a = _runs("mobilenet_v2", fused_se=False, use_graph=False)
    b = _runs("mobilenet_v2", fused_se=True, use_graph=False)
    for x, y in zip(a, b):
        _same(x, y)


# ---- block parity (DESIGN.md gate 2) ---------------------------------------------------------------
SLACK, FLOOR = 1.5, 2.5e-3


def _se_block_kinds(name):
    """index -> (block, input shape) of the first SE block of every kind (branches > 1, expansion,
    non-local, stride) of a configuration, input shapes from a CPU forward at N = 1."""
    from _cfg import build_from_cfg
    from yet_another_mobilenet_series_b200 import engine
    model, cfg = build_from_cfg(name)
    hw = cfg["flags"]["image_size"]
    shapes = {}
    hooks = [m.register_forward_hook(lambda m, i, o, k=k: shapes.__setitem__(k, tuple(i[0].shape)))
             for k, m in enumerate(model.features)]
    with torch.no_grad():
        tm_model = __import__("oracle.torch_model", fromlist=["as_reference"]).as_reference(model)
        tm_model.eval()(torch.zeros(1, 3, hw, hw))
    for hk in hooks:
        hk.remove()
    kinds = {}
    for k, m in enumerate(model.features):
        if not (hasattr(m, "expand_conv") or hasattr(m, "ops")):
            continue
        p = engine.block_parts(m)
        if p.se is None:
            continue
        kind = (len(m.channels) > 1, bool(m.expand), p.nl is not None, m.stride)
        kinds.setdefault(kind, k)
    return model, {k: shapes[k] for k in kinds.values()}


def _block_run(block, x, dy, mode):
    import copy
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200 import engine
    m = copy.deepcopy(block)
    if mode in ("fp32", "autocast"):
        m = tm.as_reference(m)
        if mode == "autocast":
            m = m.to(memory_format=torch.channels_last)
            xg = x.float().contiguous(memory_format=torch.channels_last).requires_grad_(True)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                y = m(xg)
        else:
            xg = x.float().requires_grad_(True)
            y = m(xg)
        y.float().backward(dy.float())
    else:
        engine.TRAIN_SE_FUSED = mode == "fused"
        try:
            xg = x.clone().requires_grad_(True)
            y = m(xg)
            y.backward(dy.to(y.dtype))
        finally:
            engine.TRAIN_SE_FUSED = False
    torch.cuda.synchronize()
    out = {"y": y.detach().float(), "dx": xg.grad.detach().float()}
    for n, p in m.named_parameters():
        out["grad." + n] = p.grad.detach().clone()
    for n, b in m.named_buffers():
        if "running" in n:
            out[n] = b.detach().clone()
    return out


def _gate(res, keys):
    rows, bad = [], []
    for k in keys:
        t = res["fp32"][k]
        ef, eu, ea = (_rel(res[m][k], t) for m in ("fused", "default", "autocast"))
        rows.append("%s fused %.2e default %.2e autocast %.2e" % (k, ef, eu, ea))
        # sums of a random dy that nearly cancel can put the default path itself outside the gate;
        # there the fused path must be no worse than the default (as in test_stem_train_fused_gpu)
        gate = SLACK * ea + FLOOR
        if ef > (max(gate, 1.05 * eu + 1e-4) if eu > gate else gate):
            bad.append(rows[-1])
    return rows, bad


# atomnas_c+: block 1 (no expansion), multi-branch stride 2, multi-branch stride 1; autonl_l: SE,
# SE + non-local, SE stride 2 (_se_block_kinds)
BLOCK_CASES = [(n, i) for n in ("atomnas_c+", "autonl_l") for i in range(3)]


@pytest.mark.parametrize("name,which", BLOCK_CASES)
def test_block_parity(built_lib, flags, name, which):
    """Every SE block kind of the configuration at N = 32 (case `which` of the kinds in network
    order), y / dx / every parameter gradient / every running statistic on its own."""
    from yet_another_mobilenet_series_b200 import engine
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model, kinds = _se_block_kinds(name)
    if which >= len(kinds):
        pytest.skip("%s has %d SE block kinds" % (name, len(kinds)))
    idx, shape = sorted(kinds.items())[which]
    block = model.features[idx].cuda().train()
    for mm in block.modules():
        if isinstance(mm, torch.nn.BatchNorm2d):
            with torch.no_grad():
                mm.weight.uniform_(0.5, 1.5)
                mm.running_var.uniform_(0.5, 1.5)
    N, C0, H, W = 32, shape[1], shape[2], shape[3]
    g = torch.Generator().manual_seed(idx)
    x = torch.randn(N, C0, H, W, generator=g).cuda().to(dtype=torch.bfloat16,
                                                        memory_format=torch.channels_last)
    Ho, Wo = (H - 1) // block.stride + 1, (W - 1) // block.stride + 1
    dy = torch.randn(N, block.output_dim, Ho, Wo, generator=g).cuda().to(
        memory_format=torch.channels_last)
    n0 = engine.TRAIN_SE_CALLS
    res = {m: _block_run(block, x, dy, m) for m in ("fp32", "autocast", "fused", "default")}
    assert engine.TRAIN_SE_CALLS == n0 + 1
    rows, bad = _gate(res, list(res["fp32"]))
    assert not bad, "block %d %s\n" % (idx, kinds) + "\n".join(bad + rows)


def test_stem_pair_parity(built_lib, flags):
    """AtomNAS-C+ block 1 (SE, no expansion) through the stem's fused path, where its depthwise
    backward takes the input BatchNorm (`pre`, `pre_stats`): fused_stem + fused_se against the
    fp32 graph under gate 2."""
    import copy
    from _cfg import build_from_cfg
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200 import engine, tail_ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model, cfg = build_from_cfg("atomnas_c+")
    mods = torch.nn.Sequential(model.features[0], model.features[1]).cuda().train()
    assert engine.block_parts(mods[1]).se is not None and not mods[1].expand
    hw, N = cfg["flags"]["image_size"], 32
    g = torch.Generator().manual_seed(5)
    x = torch.randn(N, 3, hw, hw, generator=g).cuda().to(dtype=torch.bfloat16,
                                                          memory_format=torch.channels_last)
    dy = torch.randn(N, mods[1].output_dim, hw // 2, hw // 2, generator=g).cuda().to(
        memory_format=torch.channels_last)
    res = {}
    for mode in ("fp32", "autocast", "fused", "default"):
        m = copy.deepcopy(mods)
        if mode in ("fp32", "autocast"):
            ref = tm.as_reference(m)
            if mode == "autocast":
                ref = ref.to(memory_format=torch.channels_last)
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    y = ref(x.float().contiguous(memory_format=torch.channels_last))
            else:
                y = ref(x.float())
            y.float().backward(dy.float())
            m = ref
        else:
            engine.TRAIN_SE_FUSED = mode == "fused"
            n0 = engine.TRAIN_SE_CALLS
            try:
                assert tail_ops.stem_block_fused_covered(m[0], m[1], x)
                y = tail_ops.stem_block_train(m[0], m[1], x)
                y.backward(dy.to(y.dtype))
            finally:
                engine.TRAIN_SE_FUSED = False
            assert engine.TRAIN_SE_CALLS == n0 + (mode == "fused")
        torch.cuda.synchronize()
        out = {"y": y.detach().float()}
        for n, p in m.named_parameters():
            out["grad." + n] = p.grad.detach().clone()
        for n, b in m.named_buffers():
            if "running" in n:
                out[n] = b.detach().clone()
        res[mode] = out
    rows, bad = _gate(res, list(res["fp32"]))
    assert not bad, "\n".join(bad + rows)


def test_partial_batch_and_calls_per_pass(built_lib, flags):
    """A partial last batch runs eagerly with fused_se, and every eager pass takes the path once
    per SE block: TRAIN_SE_CALLS rises by exactly the number of SE blocks."""
    from _cfg import build_from_cfg
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    model, cfg = build_from_cfg("autonl_l")
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    n_se = sum(1 for m in model.features if (hasattr(m, "expand_conv") or hasattr(m, "ops"))
               and engine.block_parts(m).se is not None)
    hw = cfg["flags"]["image_size"]
    ts = TrainStep(model.cuda(), 8, image_size=hw, fused_se=True)
    g = torch.Generator().manual_seed(3)
    for n in (8, 5):
        x = torch.randn(n, 3, hw, hw, generator=g).bfloat16()
        t = torch.randint(0, 1000, (n,), generator=g)
        c0 = engine.TRAIN_SE_CALLS
        loss = float(ts(x, t))
        torch.cuda.synchronize()
        assert loss == loss and 0.5 < loss < 20.0
        if n == 5 or ts.graph is None:
            assert engine.TRAIN_SE_CALLS == c0 + n_se, (n, engine.TRAIN_SE_CALLS - c0, n_se)
    assert not engine.TRAIN_SE_FUSED
