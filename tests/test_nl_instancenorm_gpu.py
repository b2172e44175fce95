"""GPU: the non-local block with `nl_norm: nn.InstanceNorm` (tracked, affine InstanceNorm2d).

1. yamb_instance_norm_fwd / _bwd against torch's F.instance_norm in fp64 (statistics, running
   statistics, dh, dgamma, dbeta; run-to-run bit equality).
2. Whole blocks against the bf16 rounding-point oracle on the tests/golden/blocks_nl_in.pt cases.
3. The AutoNL-L non-local blocks at full size against the fp32 stock-torch graph, with the
   autocast-bf16 run as the yardstick.
4. AutoNL-L built with nl_norm: nn.InstanceNorm: three TrainStep steps, eval logits, a
   bn_calibration pass, and the eval launch count."""
import copy
import os
import sys
import types

import pytest
import torch
import torch.nn.functional as F

import nl_instancenorm_oracle as no

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SLACK, FLOOR = 1.5, 2.5e-3


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _log(name, rows):
    """The measured errors (shown with pytest -s)."""
    print("\n".join(["[%s]" % name] + rows))


# ---- 1. kernels --------------------------------------------------------------------------------
def _in_fwd(h, N, HW, C, gamma, beta, rm, rv, momentum, res, res2, counter):
    from yet_another_mobilenet_series_b200 import engine, native as nat
    dev = h.device
    mean = torch.empty(N * C, device=dev)
    invstd = torch.empty(N * C, device=dev)
    y = torch.empty_like(h)
    s = nat.InFwd()
    s.N, s.HW, s.C, s.ldh = N, HW, C, C
    s.h, s.gamma, s.beta = h.data_ptr(), gamma.data_ptr(), beta.data_ptr()
    s.eps, s.momentum = 1e-3, momentum
    s.running_mean, s.running_var = rm.data_ptr(), rv.data_ptr()
    s.mean, s.invstd = mean.data_ptr(), invstd.data_ptr()
    s.residual, s.ldr, s.residual2, s.ldr2 = res.data_ptr(), C, res2.data_ptr(), C
    s.y, s.ldy = y.data_ptr(), C
    s.counter = counter.data_ptr()
    engine.launch(nat.lib().yamb_instance_norm_fwd, s)
    return y, mean.view(N, C), invstd.view(N, C)


def _in_bwd(dy, h, N, HW, C, gamma, mean, invstd, dg, db, counter):
    from yet_another_mobilenet_series_b200 import engine, native as nat
    dh = torch.empty_like(h)
    s = nat.InBwd()
    s.N, s.HW, s.C = N, HW, C
    s.ldh = s.lddy = s.lddh = C
    s.dy, s.h, s.gamma = dy.data_ptr(), h.data_ptr(), gamma.data_ptr()
    s.mean, s.invstd = mean.data_ptr(), invstd.data_ptr()
    s.dgamma, s.dbeta, s.dh = dg.data_ptr(), db.data_ptr(), dh.data_ptr()
    s.counter = counter.data_ptr()
    engine.launch(nat.lib().yamb_instance_norm_bwd, s)
    return dh


@pytest.mark.parametrize("N", [1, 3, 128])
@pytest.mark.parametrize("HW", [49, 196, 3136])
@pytest.mark.parametrize("C", [24, 40, 200, 320])
def test_kernels_vs_instance_norm(built_lib, N, HW, C):
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(N * 7 + HW + C)
    h = (torch.randn(N * HW, C, generator=g) * 2 + 3).bfloat16().to(dev)
    res = torch.randn(N * HW, C, generator=g).bfloat16().to(dev)
    res2 = torch.randn(N * HW, C, generator=g).bfloat16().to(dev)
    dy = torch.randn(N * HW, C, generator=g).bfloat16().to(dev)
    gamma = (torch.rand(C, generator=g) + 0.5).to(dev)
    beta = torch.randn(C, generator=g).to(dev)
    rm0 = torch.randn(C, generator=g).to(dev)
    rv0 = (torch.rand(C, generator=g) + 0.5).to(dev)
    counter = torch.zeros(4, device=dev, dtype=torch.int32)
    # fp64 truth on the same bf16 values
    x64 = h.double().view(N, HW, C).permute(0, 2, 1).reshape(N, C, HW, 1).requires_grad_(True)
    rm64, rv64 = rm0.double().clone(), rv0.double().clone()
    z = F.instance_norm(x64, rm64, rv64, gamma.double(), beta.double(), True, 0.1, 1e-3)
    y64 = z + (res.double() + res2.double()).view(N, HW, C).permute(0, 2, 1).reshape(N, C, HW, 1)
    dy64 = dy.double().view(N, HW, C).permute(0, 2, 1).reshape(N, C, HW, 1)
    dx64, dg64, db64 = torch.autograd.grad(z, (x64, ), dy64)[0], None, None
    xh = (x64.detach() - x64.detach().mean((2, 3), keepdim=True)) / torch.sqrt(
        x64.detach().var((2, 3), unbiased=False, keepdim=True) + 1e-3)
    dg64, db64 = (dy64 * xh).sum((0, 2, 3)), dy64.sum((0, 2, 3))
    to_nc = lambda t: t.view(N, C, HW).permute(0, 2, 1).reshape(N * HW, C)   # noqa: E731

    outs = []
    for _ in range(2):
        rm, rv = rm0.clone(), rv0.clone()
        dg = torch.full((C,), 0.25, device=dev)
        db = torch.full((C,), -0.5, device=dev)
        y, mean, invstd = _in_fwd(h, N, HW, C, gamma, beta, rm, rv, 0.1, res, res2, counter)
        dh = _in_bwd(dy, h, N, HW, C, gamma, mean, invstd, dg, db, counter)
        torch.cuda.synchronize()
        outs.append([t.clone() for t in (y, mean, invstd, rm, rv, dh, dg, db)])
    y, mean, invstd, rm, rv, dh, dg, db = outs[0]
    rows = ["N=%d HW=%d C=%d" % (N, HW, C)]
    checks = {"y": (y, to_nc(y64.detach()), 5e-3),
              "mean": (mean, x64.detach().mean((2, 3)).view(N, C), 1e-5),
              "invstd": (invstd, 1.0 / torch.sqrt(x64.detach().var((2, 3), unbiased=False)
                                                    + 1e-3).view(N, C), 1e-5),
              "running_mean": (rm, rm64, 1e-5), "running_var": (rv, rv64, 1e-5),
              "dh": (dh, to_nc(dx64), 8e-3),
              "dgamma": (dg, dg64 + 0.25, 1e-5), "dbeta": (db, db64 - 0.5, 1e-5)}
    for k, (a, b, tol) in checks.items():
        e = _rel(a, b)
        rows.append("  %-13s %.2e" % (k, e))
        assert e < tol, rows
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)                 # the same bits on every run
    assert int(counter.abs().sum()) == 0         # the arrival counter returned to zero
    # momentum None (torch passes 0): running statistics untouched
    rm, rv = rm0.clone(), rv0.clone()
    _in_fwd(h, N, HW, C, gamma, beta, rm, rv, 0.0, res, res2, counter)
    torch.cuda.synchronize()
    assert torch.equal(rm, rm0) and torch.equal(rv, rv0)
    _log("kernels", rows)


# ---- 2. blocks vs the quant oracle ------------------------------------------------------------
def _golden():
    return no.load_golden()


@pytest.mark.parametrize("name", [c[0] for c in no.CASES])
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_block_vs_quant_oracle(built_lib, name, mode):
    dev = torch.device("cuda")
    rec = _golden()[name]
    blk = no.build_block(rec)
    ref = no.build_block(rec)
    tr = mode == "train"
    cfg, P = no.extract(ref)
    yo, S = no.forward(rec["x"], cfg, P, training=tr, quant=True)
    dxo, G = no.backward(rec[mode]["dy"], cfg, P, S, training=tr, quant=True)
    blk = blk.to(dev).train(tr)
    xi = rec["x"].to(dev).requires_grad_(True)
    y = blk(xi)
    y.backward(rec[mode]["dy"].to(dev).to(y.dtype))
    torch.cuda.synchronize()
    rows = ["%s %s" % (name, mode), "  y %.2e dx %.2e" % (_rel(y.float(), yo), _rel(xi.grad, dxo))]
    assert _rel(y.float(), yo) <= 3e-3, rows
    assert _rel(xi.grad, dxo) <= 1.5e-2, rows
    grads = no.named_grads(cfg, G)
    for k, p in blk.named_parameters():
        e = _rel(p.grad.float(), grads[k].reshape(p.shape))
        rows.append("  grad %-32s %.2e" % (k, e))
        assert e <= 1.5e-2, rows
    st = dict(blk.named_buffers())
    if tr:
        assert _rel(st["nl_op.bn.running_mean"], S["bn4_rm_after"]) <= 3e-3, rows
        assert _rel(st["nl_op.bn.running_var"], S["bn4_rv_after"]) <= 3e-3, rows
    gold = rec[mode]["state_after"]
    assert int(st["nl_op.bn.num_batches_tracked"]) == int(gold["nl_op.bn.num_batches_tracked"])
    _log("blocks", rows)


# ---- 3. AutoNL-L non-local blocks at full size --------------------------------------------------
@pytest.fixture
def in_flags(monkeypatch):
    """A stand-in for the reference's utils.config whose FLAGS select the InstanceNorm."""
    mod = types.ModuleType("utils.config")
    mod.FLAGS = types.SimpleNamespace(nl_norm="nn.InstanceNorm")
    monkeypatch.setitem(sys.modules, "utils.config", mod)
    return mod


def _autonl(seed=None):
    from _cfg import build_from_cfg
    model, cfg = build_from_cfg("autonl_l", seed=seed)
    return model, cfg


def _feature_hw(model, idx):
    hw = 224
    for i, m in enumerate(model.features):
        if i == idx:
            return hw
        s = m.stride if hasattr(m, "stride") and hasattr(m, "channels") else \
            (m[0].stride[0] if isinstance(m, torch.nn.Sequential) and hasattr(m[0], "stride")
             else 1)
        hw = (hw - 1) // s + 1
    raise IndexError(idx)


@pytest.mark.parametrize("idx", [4, 9, 18, 21])
def test_autonl_block_fullsize(built_lib, in_flags, idx):
    """Gate per quantity on the mean error over two seeds: some sums are dominated by cancellation
    (features[4], seed 704: the BN1 gamma gradient is 12 % off for the BatchNorm non-local norm as
    well as for the InstanceNorm), so one draw measures the seed as much as the code."""
    from oracle import torch_model as tm
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda")
    N = 32
    model, _ = _autonl()
    hw = _feature_hw(model, idx)
    errs = {}
    rows, bad = [], []
    for seed in (700 + idx, 800 + idx):
        blk = copy.deepcopy(model.features[idx])
        assert isinstance(blk.nl_op.bn, torch.nn.InstanceNorm2d), blk
        g = torch.Generator().manual_seed(seed)
        no.randomise_norms(blk, g)
        x = torch.randn(N, blk.input_dim, hw, hw, generator=g).bfloat16().float() * 0.25
        ho = (hw - 1) // blk.stride + 1
        dy = torch.randn(N, blk.output_dim, ho, ho, generator=g).bfloat16().float()

        def run(mod, autocast):
            mod = mod.to(dev).train()
            xi = x.to(dev).requires_grad_(True)
            if autocast:
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    y = mod(xi.contiguous(memory_format=torch.channels_last))
            else:
                y = mod(xi)
            y.backward(dy.to(dev).to(y.dtype))
            torch.cuda.synchronize()
            out = {"y": y.detach().float().cpu(), "dx": xi.grad.detach().float().cpu()}
            out.update({"grad " + k: p.grad.detach().float().cpu()
                        for k, p in mod.named_parameters()})
            out.update({"stat " + k: v.detach().float().cpu()
                        for k, v in mod.named_buffers() if "running_" in k})
            return out

        truth = run(tm.as_reference(blk), False)
        yard = run(tm.as_reference(blk), True)
        ours = run(blk, False)
        for k in truth:
            errs.setdefault(k, []).append((_rel(ours[k], truth[k]), _rel(yard[k], truth[k])))
    rows.append("== AutoNL-L features[%d] N=%d %dx%d %s (mean of 2 seeds)" % (idx, N, hw, hw, blk))
    for k, es in errs.items():
        eo = sum(e[0] for e in es) / len(es)
        ea = sum(e[1] for e in es) / len(es)
        rows.append("%-40s ours %.3e  autocast %.3e" % (k, eo, ea))
        if not eo <= SLACK * ea + FLOOR:
            bad.append(rows[-1])
    _log("fullsize", rows)
    assert not bad, "\n".join(bad)


# ---- 4. the whole network -----------------------------------------------------------------------
def test_autonl_network_train_eval_calibration(built_lib, in_flags, monkeypatch):
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda")
    B = 32
    model, cfg = _autonl()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    nls = [m for m in model.modules() if isinstance(m, torch.nn.InstanceNorm2d)]
    assert nls
    fl = cfg["flags"]
    kw = dict(base_lr=fl["base_lr"], base_total_batch=fl["base_total_batch"], alpha=fl["alpha"],
              momentum=fl["momentum"], eps=fl["epsilon"], weight_decay=fl["weight_decay"],
              label_smoothing=fl["label_smoothing"], ema_decay=fl["moving_average_decay"],
              ema_base_batch=fl["moving_average_decay_base_batch"])
    ref32 = tm.RefTrainer(tm.as_reference(model).to(dev), B, **kw)
    ref16 = tm.RefTrainer(tm.as_reference(model).to(dev).to(memory_format=torch.channels_last), B,
                          autocast=torch.bfloat16, **kw)
    keys = [k for k, _ in model.named_parameters()]
    p0 = {k: v.detach().clone() for k, v in model.named_parameters()}
    model = model.to(dev)
    ts = TrainStep(model, B, image_size=fl["image_size"], **kw)
    g = torch.Generator().manual_seed(0)
    rows = ["== AutoNL-L, nl_norm nn.InstanceNorm, N=%d" % B]
    try:
        for i in range(3):
            x = torch.randn(B, 3, 224, 224, generator=g).bfloat16()
            t = torch.randint(0, 1000, (B,), generator=g)
            xd, td = x.to(dev).float(), t.to(dev)
            lt = ref32.step(xd, td) - float(tm.l2_loss_mnas(ref32.model, fl["weight_decay"]))
            la = ref16.step(xd.contiguous(memory_format=torch.channels_last), td) - \
                float(tm.l2_loss_mnas(ref16.model, fl["weight_decay"]))
            lo = float(ts(x, t))
            rows.append("step %d loss ours %.5f fp32 %.5f autocast %.5f" % (i, lo, lt, la))
            assert abs(lo - lt) <= 2.0 * abs(la - lt) + 5e-3 * abs(lt), rows
        torch.cuda.synchronize()
        assert ts.graph is not None
        flat = lambda d: torch.cat([d[k].detach().double().flatten().cpu() for k in keys])  # noqa
        p0f = flat(p0)
        eo = _rel(flat(dict(model.named_parameters())) - p0f,
                  flat(dict(ref32.model.named_parameters())) - p0f)
        ea = _rel(flat(dict(ref16.model.named_parameters())) - p0f,
                  flat(dict(ref32.model.named_parameters())) - p0f)
        rows.append("update rel-L2 ours %.4f autocast %.4f" % (eo, ea))
        assert eo <= 1.3 * ea + 1e-2, rows
        bo, bt, ba = (dict(m.named_buffers()) for m in (model, ref32.model, ref16.model))
        for kind in ("running_mean", "running_var"):
            ks = [k for k in bt if k.endswith(kind) and k.rpartition(".")[0].endswith("nl_op.bn")]
            mo = sum(_rel(bo[k], bt[k]) for k in ks) / len(ks)
            ma = sum(_rel(ba[k], bt[k]) for k in ks) / len(ks)
            rows.append("InstanceNorm %s mean rel-L2 ours %.2e autocast %.2e" % (kind, mo, ma))
            assert mo <= 1.5 * ma + 2e-3, rows
        for k in bt:
            if k.endswith("nl_op.bn.num_batches_tracked"):
                assert int(bo[k]) == int(bt[k]) == 0      # InstanceNorm never counts batches

        # ---- eval logits: default dispatch and the four-launch sequence, vs fp32 truth ----
        model.eval()
        ref32.model.load_state_dict(model.state_dict())
        ref16.model.load_state_dict(model.state_dict())
        ref32.model.eval()
        ref16.model.eval()
        xe = torch.randn(B, 3, 224, 224, generator=g).bfloat16().to(dev)
        with torch.no_grad():
            truth = ref32.model(xe.float()).float()
            with torch.autocast("cuda", dtype=torch.bfloat16):
                yard = ref16.model(xe.float().contiguous(memory_format=torch.channels_last)).float()
            n0 = engine.EVAL_FUSED_CALLS
            l0 = engine.LAUNCHES
            ours = model(xe).float()
            launches_in = engine.LAUNCHES - l0
            assert engine.EVAL_FUSED_CALLS > n0          # the fused-class eval path was taken
            monkeypatch.setattr(engine, "EVAL_FUSED", False)
            ours4 = model(xe).float()
            monkeypatch.setattr(engine, "EVAL_FUSED", True)
        ea = _rel(yard, truth)
        for tag, o in (("default", ours), ("YAMB_EVAL_FUSED=0", ours4)):
            eo = _rel(o, truth)
            rows.append("eval logits (%s) ours %.3e autocast %.3e" % (tag, eo, ea))
            assert eo <= SLACK * ea + FLOOR, rows

        # ---- the same network with the BatchNorm non-local norm: same eval launch count ----
        in_flags.FLAGS = types.SimpleNamespace()          # FLAGS without nl_norm: ZeroInitBN
        bn_model, _ = _autonl()
        assert not any(isinstance(m, torch.nn.InstanceNorm2d) for m in bn_model.modules())
        bn_model = bn_model.to(dev).eval()
        with torch.no_grad():
            l0 = engine.LAUNCHES
            bn_model(xe)
            launches_bn = engine.LAUNCHES - l0
        rows.append("eval launches: InstanceNorm %d BatchNorm %d" % (launches_in, launches_bn))
        assert launches_in == launches_bn, rows

        # ---- bn_calibration (reference utils/common.py:175-187): BatchNorms re-estimate their
        #      statistics cumulatively in train mode, the InstanceNorms stay in eval mode ----
        def bn_calibration(m, cumulative_bn_stats=True):
            if isinstance(m, torch.nn.BatchNorm2d):
                m.reset_running_stats()
                m.train()
                if cumulative_bn_stats:
                    m.momentum = None

        ref = tm.as_reference(model)
        ref_a = tm.as_reference(model).to(memory_format=torch.channels_last)
        for m in (model, ref, ref_a):
            m.apply(bn_calibration)
        assert all(not m.training for m in nls)
        with torch.no_grad():
            for _ in range(2):
                xc = torch.randn(B, 3, 224, 224, generator=g).bfloat16().to(dev)
                model(xc)
                ref(xc.float())
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    ref_a(xc.float().contiguous(memory_format=torch.channels_last))
        torch.cuda.synchronize()
        bo, bt, ba = (dict(m.named_buffers()) for m in (model, ref, ref_a))
        ks = [k for k in bt if "running_" in k]
        mo = sum(_rel(bo[k], bt[k]) for k in ks) / len(ks)
        ma = sum(_rel(ba[k], bt[k]) for k in ks) / len(ks)
        rows.append("bn_calibration running statistics: mean rel-L2 ours %.2e autocast %.2e"
                    % (mo, ma))
        assert mo <= SLACK * ma + FLOOR, rows
        for k in bt:
            if k.endswith("num_batches_tracked"):
                assert int(bo[k]) == int(bt[k]), k
    finally:
        _log("network", rows)
