"""GPU: the training-mode expand + depthwise forward from x (yamb_expand_dw_train_fwd,
TrainStep(fused_expand_dw=True)).

- Every compiled instantiation (k, stride, tile plan, clamp / generic activation) on odd N, maps
  that do not divide into tiles, a partial last 64-channel slice and Cin padded to 16: z2 bitwise
  yamb_depthwise_fwd's on the pointwise GEMM's h1 with the same BatchNorm-1 coefficients; z2
  within bf16 rounding of an fp64 stencil; BatchNorm-2 mean, invstd and running statistics within
  1e-6 of fp64 (plus the bf16 rounding of the activated input), and within 1e-6 of
  yamb_depthwise_fwd's.
- Block forward + backward of every covered MobileNetV2, Proxyless and AutoNL-L block kind with the
  switch on and off: bitwise equal, or (where BatchNorm-2's summation order moves a last bit) both
  within the autocast yardstick of the fp32 reference.
- Three TrainStep(fused_expand_dw=True) steps against the fp32 reference step; graph replay gives
  eager's bits, two runs give the same bits, and the path is taken."""
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


@pytest.fixture
def all_shapes(monkeypatch):
    """Every covered block takes the path (the shape rule off)."""
    from yet_another_mobilenet_series_b200 import engine
    monkeypatch.setattr(engine, "EXPAND_DW_SHAPE_RULE", False)


def _call(fn, a):
    from yet_another_mobilenet_series_b200 import native as nat
    nat.check(fn(C.byref(a), nat.stream_handle()))


class _Bn2:
    """A yamb_bn_fwd with its own workspace, gamma / beta and running statistics."""

    def __init__(self, Cc, count, g, momentum=0.1, eps=1e-3):
        from yet_another_mobilenet_series_b200 import native as nat
        self.partials = torch.zeros(2 * Cc, dtype=torch.float64, device="cuda")
        self.counter = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.gamma = (torch.rand(Cc, generator=g) + 0.5).cuda()
        self.beta = (torch.rand(Cc, generator=g) - 0.5).cuda()
        self.rm = (torch.rand(Cc, generator=g) - 0.5).cuda()
        self.rv = (torch.rand(Cc, generator=g) + 0.5).cuda()
        self.rm0, self.rv0 = self.rm.clone(), self.rv.clone()
        self.nbt = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.scale, self.shift, self.mean, self.invstd = (torch.zeros(Cc, device="cuda")
                                                          for _ in range(4))
        self.momentum, self.eps, self.count = momentum, eps, count
        s = nat.BnFwd()
        s.partials, s.counter = self.partials.data_ptr(), self.counter.data_ptr()
        s.gamma, s.beta, s.eps, s.momentum = self.gamma.data_ptr(), self.beta.data_ptr(), eps, momentum
        s.running_mean, s.running_var = self.rm.data_ptr(), self.rv.data_ptr()
        s.num_batches_tracked = self.nbt.data_ptr()
        s.scale, s.shift = self.scale.data_ptr(), self.shift.data_ptr()
        s.mean, s.invstd = self.mean.data_ptr(), self.invstd.data_ptr()
        s.count = count
        self.s = s


def _act64(z, act):
    if act == 1:
        return z.clamp_min(0)
    if act == 2:
        return z.clamp(0, 6)
    if act == 3:
        return z * torch.sigmoid(z)
    return z * (z + 3).clamp(0, 6) / 6


# (k, stride, N, H, W, Cin, Chid): each selects one tile plan of (k, stride) — stride 1, k = 3 / 5:
# 7x16 on the 15-wide maps, two 7x7 images per tile on the 7x7 maps — with odd N, maps that do not
# divide into tiles, a partial last 64-channel slice (Chid % 64 != 0) and Cin padded to 16
GEOMS = [(3, 1, 3, 15, 15, 24, 144), (3, 1, 3, 7, 7, 40, 96), (3, 2, 3, 15, 17, 32, 200),
         (5, 1, 3, 15, 13, 40, 240), (5, 1, 5, 7, 7, 80, 480), (5, 2, 3, 15, 15, 24, 72),
         (7, 1, 3, 15, 13, 48, 288), (7, 2, 3, 29, 29, 16, 96), (3, 1, 2, 9, 9, 256, 520),
         (3, 2, 3, 8, 8, 8, 40)]
# every geometry with a clamp activation (ReLU / ReLU6) and a generic one (Swish / h-swish)
CASES = [g + (a,) for i, g in enumerate(GEOMS) for a in ((1, 3) if i % 2 else (2, 4))]


@pytest.mark.parametrize("k,s,N,H,W,Cin,Chid,act", CASES)
def test_kernel_vs_depthwise_and_fp64(built_lib, k, s, N, H, W, Cin, Chid, act):
    from yet_another_mobilenet_series_b200 import native as nat
    lib = nat.lib()
    g = torch.Generator().manual_seed(k * 1000 + s * 100 + Cin + Chid + act)
    M = N * H * W
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    Mo = N * Ho * Wo
    x = torch.randn(M, Cin, generator=g).to(torch.bfloat16).cuda()
    w1 = (torch.randn(Chid, Cin, generator=g) / Cin ** 0.5).to(torch.bfloat16).cuda()
    s1 = (torch.rand(Chid, generator=g) + 0.5).cuda()
    t1 = (torch.rand(Chid, generator=g) - 0.5).cuda()
    wdw = (torch.randn(Chid, 1, k, k, generator=g) / k).cuda()
    # the expand GEMM's h1
    h1 = torch.empty(M, Chid, dtype=torch.bfloat16, device="cuda")
    gm = nat.Gemm()
    gm.M, gm.N, gm.K = M, Chid, Cin
    gm.A, gm.lda, gm.B, gm.ldb, gm.D, gm.ldd = x.data_ptr(), Cin, w1.data_ptr(), Cin, h1.data_ptr(), Chid
    _call(lib.yamb_pointwise_gemm, gm)
    # the default step 2: yamb_depthwise_fwd on h1 with BatchNorm 1 + act on load
    z_ref = torch.full((Mo, Chid), float("nan"), dtype=torch.bfloat16, device="cuda")
    bn_ref = _Bn2(Chid, Mo, torch.Generator().manual_seed(5))
    d = nat.DwFwd()
    d.N, d.H, d.W, d.C, d.ldc, d.k, d.stride = N, H, W, Chid, Chid, k, s
    d.x, d.w, d.y = h1.data_ptr(), wdw.data_ptr(), z_ref.data_ptr()
    d.in_scale, d.in_shift, d.in_act = s1.data_ptr(), t1.data_ptr(), act
    d.bn = C.pointer(bn_ref.s)
    _call(lib.yamb_depthwise_fwd, d)
    # the fused kernel, twice (the statistics workspace returns to zero; same z2 bits)
    outs = []
    for _ in range(2):
        z = torch.full((Mo, Chid), float("nan"), dtype=torch.bfloat16, device="cuda")
        bn = _Bn2(Chid, Mo, torch.Generator().manual_seed(5))
        a = nat.ExpandDwTrain()
        a.N, a.H, a.W, a.Cin, a.Chid, a.kernel, a.stride, a.act, a.ldh = N, H, W, Cin, Chid, k, s, act, Chid
        a.x, a.w_expand, a.bn1_scale, a.bn1_shift = x.data_ptr(), w1.data_ptr(), s1.data_ptr(), t1.data_ptr()
        a.w_dw, a.h2, a.bn = wdw.data_ptr(), z.data_ptr(), C.pointer(bn.s)
        _call(lib.yamb_expand_dw_train_fwd, a)
        torch.cuda.synchronize()
        assert int(bn.counter.item()) == 0 and not bool(bn.partials.any())
        outs.append((z, bn))
    z, bn = outs[0]
    assert torch.equal(z.view(torch.int16), z_ref.view(torch.int16)), \
        "z2 differs from depthwise_fwd at %d of %d elements" % (
            int((z.view(torch.int16) != z_ref.view(torch.int16)).sum()), z.numel())
    assert torch.equal(outs[1][0].view(torch.int16), z.view(torch.int16))
    # fp64 stencil of the activated input (its bf16 rounding and z2's bound the difference)
    a1 = _act64(h1.double() * s1.double() + t1.double(), act)
    a1n = a1.view(N, H, W, Chid).permute(0, 3, 1, 2)
    z64 = torch.nn.functional.conv2d(a1n, wdw.double(), stride=s, padding=(k - 1) // 2, groups=Chid)
    zabs = torch.nn.functional.conv2d(a1n.abs(), wdw.double().abs(), stride=s, padding=(k - 1) // 2,
                                      groups=Chid)
    z64 = z64.permute(0, 2, 3, 1).reshape(Mo, Chid)
    zabs = zabs.permute(0, 2, 3, 1).reshape(Mo, Chid)
    bound = zabs * (2.0 ** -8 + 2e-6) + z64.abs() * 2.0 ** -8 + 1e-6
    err = (z.double() - z64).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    # BatchNorm 2 against fp64 statistics of the fp64 stencil (tolerance: 1e-6 plus the effect of
    # rounding the activated input to bf16): mean and invstd, running statistics with the
    # unbiased variance
    mean64, var64 = z64.mean(0), z64.var(0, unbiased=False)
    rms = (z64 * z64).mean(0).sqrt()
    tol = 1e-6 + zabs.mean(0) * 2.0 ** -8 / rms.clamp_min(1e-30)   # a1's bf16 rounding
    assert bool(((bn.mean.double() - mean64).abs() <= tol * rms).all())
    inv64 = 1.0 / (var64 + bn.eps).sqrt()
    assert bool(((bn.invstd.double() - inv64).abs() <= 2 * tol * inv64).all())
    m = bn.momentum
    rm64 = (1 - m) * bn.rm0.double() + m * mean64
    rv64 = (1 - m) * bn.rv0.double() + m * z64.var(0, unbiased=True)
    assert bool(((bn.rm.double() - rm64).abs() <= tol * (rms + bn.rm0.double().abs())).all())
    assert bool(((bn.rv.double() - rv64).abs() <= 2 * tol * rv64).all())
    assert int(bn.nbt.item()) == 1
    # against the default step's statistics of the same z2 (two fixed-order fp32 / double sums)
    assert bool(((bn.mean - bn_ref.mean).abs() <= 1e-6 * rms.float()).all())
    assert torch.allclose(bn.invstd, bn_ref.invstd, rtol=1e-6, atol=0)
    assert torch.allclose(bn.scale, bn_ref.scale, rtol=1e-6, atol=0)


# ---- block forward + backward ---------------------------------------------------------------------
def _rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def _covered_kinds(name):
    """index -> input shape of the first covered block of every (k, stride, H) of a configuration,
    input shapes from a CPU forward at N = 1."""
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
        kind = engine.expand_dw_kind(m, shapes[k][2], shapes[k][3])
        if kind is not None:
            kinds.setdefault(kind[:3], k)
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
        engine.TRAIN_EXPAND_DW_FUSED = mode == "fused"
        try:
            xg = x.clone().requires_grad_(True)
            y = m(xg)
            y.backward(dy.to(y.dtype))
        finally:
            engine.TRAIN_EXPAND_DW_FUSED = False
    torch.cuda.synchronize()
    out = {"y": y.detach().float(), "dx": xg.grad.detach().float()}
    for n, p in m.named_parameters():
        out["grad." + n] = p.grad.detach().clone()
    for n, b in m.named_buffers():
        if "running" in n:
            out[n] = b.detach().clone()
    return out


SLACK, FLOOR = 1.5, 2.5e-3
# covered block kinds (k, stride, input size) per configuration
KIND_COUNTS = (("mobilenet_v2", 8), ("proxyless_mobile", 9), ("autonl_l", 10))
BLOCK_CASES = [(n, i) for n, c in KIND_COUNTS for i in range(c)]


@pytest.mark.parametrize("name,which", BLOCK_CASES)
def test_block_on_off(built_lib, flags, all_shapes, name, which):
    """Covered block kind `which` (k, stride, input size; network order) at N = 32: y, dx, every
    parameter gradient and every running statistic bitwise equal with the switch on and off, or,
    where BatchNorm-2's summation order moves a bit, both within the autocast yardstick of fp32."""
    from yet_another_mobilenet_series_b200 import engine
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model, kinds = _covered_kinds(name)
    assert len(kinds) == dict(KIND_COUNTS)[name]
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
    n0 = engine.TRAIN_EXPAND_DW_CALLS
    fused = _block_run(block, x, dy, "fused")
    assert engine.TRAIN_EXPAND_DW_CALLS == n0 + 1
    default = _block_run(block, x, dy, "default")
    assert engine.TRAIN_EXPAND_DW_CALLS == n0 + 1
    differ = [k for k in default if not torch.equal(fused[k], default[k])]
    if not differ:
        return
    res = {"fused": fused, "default": default,
           "fp32": _block_run(block, x, dy, "fp32"), "autocast": _block_run(block, x, dy, "autocast")}
    rows, bad = [], []
    for k in differ:
        t = res["fp32"][k]
        ef, eu, ea = (_rel(res[m][k], t) for m in ("fused", "default", "autocast"))
        rows.append("%s fused %.2e default %.2e autocast %.2e" % (k, ef, eu, ea))
        gate = SLACK * ea + FLOOR
        if ef > (max(gate, 1.05 * eu + 1e-4) if eu > gate else gate):
            bad.append(rows[-1])
    assert not bad, "block %d\n" % idx + "\n".join(bad + rows)


# ---- TrainStep(fused_expand_dw=True) --------------------------------------------------------------
def _flat(d, keys):
    return torch.cat([d[k].detach().double().flatten().cpu() for k in keys])


@pytest.mark.parametrize("name", ["mobilenet_v2", "proxyless_mobile", "autonl_l", "atomnas_c+"])
def test_three_steps_vs_fp32_reference(built_lib, flags, all_shapes, name):
    """The rule of test_configs_gpu / test_se_train_fused_gpu: losses within twice the autocast
    step's distance from the fp32 step, updates and running statistics within its error.
    AtomNAS-C+ has no single-branch block with expansion: the switch changes nothing there."""
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
    ts = TrainStep(model, B, image_size=hw, fused_expand_dw=True, **kw)
    g = torch.Generator().manual_seed(0)
    keys = [k for k, _ in model.named_parameters()]
    n0 = engine.TRAIN_EXPAND_DW_CALLS
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
    assert (engine.TRAIN_EXPAND_DW_CALLS > n0) == (name != "atomnas_c+")
    assert not engine.TRAIN_EXPAND_DW_FUSED
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


def test_graph_replay_equals_eager_and_runs_repeat(built_lib, flags, all_shapes):
    from yet_another_mobilenet_series_b200 import engine
    n0 = engine.TRAIN_EXPAND_DW_CALLS
    runs = [_runs("mobilenet_v2", fused_expand_dw=True, use_graph=ug) for ug in (False, True, True)]
    assert engine.TRAIN_EXPAND_DW_CALLS > n0
    for a, b, c in zip(*runs):
        _same(a, b)
        _same(b, c)


def test_combined_switches_and_partial_batch(built_lib, flags, all_shapes):
    """With fused_stem, fused_tail, fused_se and micro_batch, and on a partial last batch (eager),
    every eager pass takes the path once per covered block."""
    from _cfg import build_from_cfg
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    model, cfg = build_from_cfg("autonl_l")
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    hw = cfg["flags"]["image_size"]
    n_cov = sum(1 for m in model.features if (hasattr(m, "expand_conv") or hasattr(m, "ops"))
                and engine.expand_dw_kind(m, 1, 1) is not None)
    ts = TrainStep(model.cuda(), 8, image_size=hw, fused_expand_dw=True, fused_stem=True,
                   fused_tail=True, fused_se=True, micro_batch=4, use_graph=False)
    g = torch.Generator().manual_seed(3)
    for n, passes in ((8, 2), (5, 2)):
        x = torch.randn(n, 3, hw, hw, generator=g).bfloat16()
        t = torch.randint(0, 1000, (n,), generator=g)
        c0 = engine.TRAIN_EXPAND_DW_CALLS
        loss = float(ts(x, t))
        torch.cuda.synchronize()
        assert loss == loss and 0.5 < loss < 20.0
        assert engine.TRAIN_EXPAND_DW_CALLS == c0 + passes * n_cov, (n, engine.TRAIN_EXPAND_DW_CALLS - c0)
    assert not engine.TRAIN_EXPAND_DW_FUSED
