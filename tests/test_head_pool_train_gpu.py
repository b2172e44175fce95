"""GPU: the training-mode head kernels (yamb_head_pool_train_fwd / _bwd, csrc/head_train.cu) and
`TrainStep(fused_tail=True)`.

1. Both kernels, called directly, against a float64 restatement built from the same bf16 h, element
   by element, for every activation, C in {8, 1280, 1792} and HW in {49, 1, 63 (7x9)} with odd N
   (pixel chunks and 256-lane groups that do not divide evenly).  u = 2^-24.
   pooled: a = bf16(act(fmaf(scale, h, shift))) restated in fp64 (z exact to fp32 rounding);
     |pooled - mean(a64)| <= 1 bf16 ulp + the fp32 sum's HW u mean|a| (+ 1 bf16 ulp of a for the
     Swish / h-swish intrinsics).
   sum(dz), sum(dz xhat) (read back as dbeta, dgamma, accumulated onto non-zero values): within
     1e-5 of the sums of |terms|, the fp32 per-thread chains being short (<= 64 terms here).
   ca, cb, cc: the fp64 finalize of those sums, within 1e-4 relative of their terms.
   dh: the value the kernel rounds, ca dz + cb h + cc with the kernel's own coefficients in fp64,
     must round to within 1 bf16 ulp of the stored bf16 (+ 4u of the terms).
2. The fused head (GEMM + fused pool) and the unfused one against the fp32 head in torch, under
   the autocast yardstick of DESIGN.md §c gate 2: pooled, dx, dW, dgamma, dbeta and the running
   statistics; the running statistics are bitwise those of the unfused head (the GEMM takes them).
3. Two runs, and eager against CUDA-graph replay, give the same bits.
4. TrainStep(fused_tail=True) on MobileNetV2-1.0 and AutoNL-L (Swish head), N = 16: three steps
   against the reference step sequence in fp32 with the rule of tests/test_configs_gpu.py; with
   micro_batch; a checkpoint written with the flag resumes bit-exactly with it."""
import ctypes as C
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
ACTS = {0: "Identity", 1: "ReLU", 2: "ReLU6", 3: "Swish", 4: "HSwish"}


def _ulp_bf16(x):
    x = np.maximum(np.abs(x), 2.0 ** -126)
    return 2.0 ** (np.floor(np.log2(x)) - 7)


def _act64(z, act):
    if act == 1:
        return np.maximum(z, 0)
    if act == 2:
        return np.clip(z, 0, 6)
    if act == 3:
        return z / (1 + np.exp(-z))
    if act == 4:
        return z * np.clip(z + 3, 0, 6) / 6
    return z


def _dact64(z, act):
    if act == 1:
        return (z > 0).astype(np.float64)
    if act == 2:
        return ((z > 0) & (z < 6)).astype(np.float64)
    if act == 3:
        s = 1 / (1 + np.exp(-z))
        return s * (1 + z * (1 - s))
    if act == 4:
        return np.where(z <= -3, 0.0, np.where(z >= 3, 1.0, (2 * z + 3) / 6))
    return np.ones_like(z)


def _bf16_np(t):
    return t.float().cpu().double().numpy()


def _case(N, HW, Cc, act, seed):
    from yet_another_mobilenet_series_b200 import engine
    g = torch.Generator().manual_seed(seed)
    dev = torch.device("cuda")
    h = (torch.randn(N * HW, Cc, generator=g) * 1.3 + 0.2).bfloat16()
    mean = h.float().mean(0)
    var = h.float().var(0, unbiased=False)
    invstd = torch.rsqrt(var + 1e-5)
    gamma = torch.rand(Cc, generator=g) + 0.5
    beta = torch.randn(Cc, generator=g) * 0.5
    scale = gamma * invstd
    shift = beta - mean * scale
    dp = (torch.randn(N, Cc, generator=g) * 0.1).bfloat16()
    d = {k: v.to(dev) for k, v in dict(h=h, mean=mean, invstd=invstd, gamma=gamma, scale=scale,
                                        shift=shift, dp=dp).items()}
    d["dgamma0"] = (torch.randn(Cc, generator=g) * 1e-3).to(dev)
    d["dbeta0"] = (torch.randn(Cc, generator=g) * 1e-3).to(dev)
    d["ws"] = engine.Workspace.get(dev)
    return d


def _fwd(lib, d, N, HW, Cc, act):
    from yet_another_mobilenet_series_b200 import native as nat
    pooled = torch.empty(N, Cc, device="cuda", dtype=torch.bfloat16)
    a = nat.HeadPoolTrain()
    a.N, a.HW, a.C, a.act = N, HW, Cc, act
    a.h, a.scale, a.shift, a.pooled = (d["h"].data_ptr(), d["scale"].data_ptr(),
                                       d["shift"].data_ptr(), pooled.data_ptr())
    nat.check(lib.yamb_head_pool_train_fwd(C.byref(a), nat.stream_handle()))
    return pooled


def _bwd(lib, d, N, HW, Cc, act):
    from yet_another_mobilenet_series_b200 import native as nat
    o = {k: torch.zeros(Cc, device="cuda") for k in ("ca", "cb", "cc")}
    o["dgamma"], o["dbeta"] = d["dgamma0"].clone(), d["dbeta0"].clone()
    o["dh"] = torch.empty(N * HW, Cc, device="cuda", dtype=torch.bfloat16)
    a = nat.HeadPoolTrainGrad()
    a.N, a.HW, a.C, a.act = N, HW, Cc, act
    a.h, a.scale, a.shift = d["h"].data_ptr(), d["scale"].data_ptr(), d["shift"].data_ptr()
    a.dpooled, a.dh = d["dp"].data_ptr(), o["dh"].data_ptr()
    b = a.bn
    b.partials, b.counter = d["ws"].stats(Cc)
    b.gamma, b.mean, b.invstd = d["gamma"].data_ptr(), d["mean"].data_ptr(), d["invstd"].data_ptr()
    b.dgamma, b.dbeta = o["dgamma"].data_ptr(), o["dbeta"].data_ptr()
    b.ca, b.cb, b.cc = o["ca"].data_ptr(), o["cb"].data_ptr(), o["cc"].data_ptr()
    b.count, b.use_batch_stats = N * HW, 1
    nat.check(lib.yamb_head_pool_train_bwd(C.byref(a), nat.stream_handle()))
    return o


def _bad(what, got, want, tol):
    bad = np.argwhere(~(np.abs(got - want) <= tol))
    return "%s: %d bad, first %s got %r want %r tol %r" % (
        what, len(bad), bad[:3].tolist(), got[tuple(bad[0])] if len(bad) else None,
        want[tuple(bad[0])] if len(bad) else None, tol[tuple(bad[0])] if len(bad) else None)


KERNEL_CASES = [(N, HW, Cc, act) for Cc in (8, 1280, 1792) for (N, HW) in ((5, 49), (3, 1), (7, 63))
                for act in ACTS]


@pytest.mark.parametrize("N,HW,Cc,act", KERNEL_CASES)
def test_kernels_vs_fp64(built_lib, N, HW, Cc, act):
    d = _case(N, HW, Cc, act, seed=N * 1000 + HW * 10 + act + Cc)
    pooled = _fwd(built_lib, d, N, HW, Cc, act)
    o = _bwd(built_lib, d, N, HW, Cc, act)
    torch.cuda.synchronize()
    h = _bf16_np(d["h"])
    sc, sh = (d[k].cpu().double().numpy() for k in ("scale", "shift"))
    mu, rs, gam = (d[k].cpu().double().numpy() for k in ("mean", "invstd", "gamma"))
    z = (sc * h + sh).astype(np.float32).astype(np.float64)       # fmaf: one fp32 rounding
    intr = act in (3, 4)
    # ---- forward ----
    a = torch.from_numpy(_act64(z, act)).bfloat16().double().numpy().reshape(N, HW, Cc)
    p64 = a.mean(1)
    tol = _ulp_bf16(p64) + HW * U * np.abs(a).mean(1) + 1e-30
    if intr:
        tol = tol + _ulp_bf16(np.abs(a)).mean(1)
    got = _bf16_np(pooled)
    assert np.all(np.abs(got - p64) <= tol), _bad("pooled", got, p64, tol)
    # ---- backward sums and coefficients ----
    dy = (_bf16_np(d["dp"]) * np.float32(1.0 / HW)).astype(np.float32).astype(np.float64)
    dz = np.repeat(dy, HW, axis=0) * _dact64(z, act)
    xhat = (h - mu) * rs
    S, Q = dz.sum(0), (dz * xhat).sum(0)
    tS = 1e-5 * np.abs(dz).sum(0) + 1e-30
    tQ = 1e-5 * np.abs(dz * xhat).sum(0) + 1e-30
    db0, dg0 = d["dbeta0"].cpu().double().numpy(), d["dgamma0"].cpu().double().numpy()
    got_db = o["dbeta"].cpu().double().numpy()
    got_dg = o["dgamma"].cpu().double().numpy()
    assert np.all(np.abs(got_db - (db0 + S)) <= tS + U * np.abs(db0 + S)), _bad(
        "sum dz", got_db, db0 + S, tS)
    assert np.all(np.abs(got_dg - (dg0 + Q)) <= tQ + U * np.abs(dg0 + Q)), _bad(
        "sum dz xhat", got_dg, dg0 + Q, tQ)
    cnt = N * HW
    scg = gam * rs
    m1, m2 = S / cnt, Q / cnt
    ca64, cb64, cc64 = scg, -scg * rs * m2, scg * (mu * rs * m2 - m1)
    ca, cb, cc = (o[k].cpu().double().numpy() for k in ("ca", "cb", "cc"))
    assert np.all(np.abs(ca - ca64) <= 4 * U * np.abs(ca64)), _bad("ca", ca, ca64, 4 * U * np.abs(ca64))
    tcb = 1e-4 * np.abs(cb64) + np.abs(scg * rs) * tQ / cnt
    assert np.all(np.abs(cb - cb64) <= tcb), _bad("cb", cb, cb64, tcb)
    tcc = 1e-4 * np.abs(scg) * (np.abs(mu * rs * m2) + np.abs(m1)) + np.abs(scg) * (
        np.abs(mu * rs) * tQ + tS) / cnt + 1e-30
    assert np.all(np.abs(cc - cc64) <= tcc), _bad("cc", cc, cc64, tcc)
    # ---- dh: the value the kernel rounds, from its own coefficients ----
    pre = ca * dz + cb * h + cc
    terms = np.abs(ca * dz) + np.abs(cb * h) + np.abs(cc)
    tol = _ulp_bf16(pre) + 4 * U * terms + (4e-6 * np.abs(ca * dz) if intr else 0) + 1e-30
    got = _bf16_np(o["dh"])
    assert np.all(np.abs(got - pre) <= tol), _bad("dh", got, pre, tol)


def test_kernels_same_bits_twice_and_in_a_graph(built_lib):
    N, HW, Cc, act = 9, 49, 1280, 3
    d = _case(N, HW, Cc, act, seed=7)
    runs = []
    for _ in range(2):
        p = _fwd(built_lib, d, N, HW, Cc, act)
        runs.append([p] + [v for _, v in sorted(_bwd(built_lib, d, N, HW, Cc, act).items())])
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        d = _ws_of_stream(d)              # the statistics workspace of the capturing stream
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            p = _fwd(built_lib, d, N, HW, Cc, act)
            o = _bwd(built_lib, d, N, HW, Cc, act)
    g.replay()
    torch.cuda.synchronize()
    runs.append([p] + [v for _, v in sorted(o.items())])
    for r in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(runs[0], r))


def _ws_of_stream(d):
    from yet_another_mobilenet_series_b200 import engine
    d = dict(d)
    d["ws"] = engine.Workspace.get(torch.device("cuda"))
    return d


# ---- the head module, fused against unfused and the fp32 truth -------------------------------------
def _head(act_name, Cin, Cout, seed):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    torch.manual_seed(seed)
    head = mb.ConvBNReLU(Cin, Cout, kernel_size=1, active_fn=mb.get_active_fn(act_name),
                         batch_norm_kwargs={"momentum": 0.1, "eps": 1e-5})
    head.apply(mb.init_weights_mnas)
    with torch.no_grad():
        head[1].weight.uniform_(0.5, 1.5)
        head[1].bias.normal_(0, 0.3)
    return head


def _run_head(head, x, dp, mode):
    """(pooled, dx, dW, dgamma, dbeta, running_mean, running_var) of one training forward +
    backward; mode 'fused', 'unfused' (this package), 'fp32' / 'autocast' (stock torch)."""
    from yet_another_mobilenet_series_b200 import engine, tail_ops
    from oracle import torch_model as tm
    import copy
    m = copy.deepcopy(head).cuda().train()
    xg = x.clone().cuda().requires_grad_(True)
    if mode in ("fp32", "autocast"):
        m = tm.as_reference(m)
        if mode == "autocast":
            m = m.to(memory_format=torch.channels_last)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode == "autocast"):
            xin = xg.contiguous(memory_format=torch.channels_last) if mode == "autocast" else xg
            pooled = m(xin).mean((2, 3))
    elif mode == "fused":
        engine.TRAIN_TAIL_FUSED = True
        try:
            n0 = engine.TRAIN_TAIL_CALLS
            pooled = tail_ops.head_pool_train(m, xg).flatten(1)
            assert engine.TRAIN_TAIL_CALLS == n0 + 1
        finally:
            engine.TRAIN_TAIL_FUSED = False
    else:
        pooled = m(xg).mean((2, 3))
    pooled.backward(dp.cuda().to(pooled.dtype))
    torch.cuda.synchronize()
    return [t.detach().double().cpu() for t in (
        pooled, xg.grad, m[0].weight.grad, m[1].weight.grad, m[1].bias.grad, m[1].running_mean,
        m[1].running_var)]


NAMES = ("pooled", "dx", "dW", "dgamma", "dbeta", "running_mean", "running_var")


@pytest.mark.parametrize("act_name,Cin,Cout,N,hw", [("nn.ReLU6", 320, 1280, 32, 7),
                                                    ("nn.Swish", 384, 1280, 17, 7),
                                                    ("nn.ReLU", 448, 1792, 9, 5)])
def test_fused_head_vs_fp32_truth(built_lib, act_name, Cin, Cout, N, hw):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    head = _head(act_name, Cin, Cout, seed=Cout + N)
    g = torch.Generator().manual_seed(N)
    x = torch.randn(N, Cin, hw, hw, generator=g).bfloat16().float()
    dp = torch.randn(N, Cout, generator=g) * 0.05
    out = {m: _run_head(head, x, dp, m) for m in ("fused", "unfused", "fp32", "autocast")}
    rel = lambda a, b: float((a - b).norm() / (b.norm() + 1e-30))
    rows = []
    for i, name in enumerate(NAMES):
        t = out["fp32"][i]
        ef, eu, ea = rel(out["fused"][i], t), rel(out["unfused"][i], t), rel(out["autocast"][i], t)
        rows.append("%s fused %.2e unfused %.2e autocast %.2e" % (name, ef, eu, ea))
        assert ef <= 1.5 * ea + 2.5e-3, rows
    for i in (5, 6):               # the head GEMM's epilogue takes the statistics either way
        assert torch.equal(out["fused"][i], out["unfused"][i]), NAMES[i]


# ---- TrainStep(fused_tail=True) ------------------------------------------------------------------
@pytest.fixture
def flags(monkeypatch):
    """A stand-in for the reference's utils.config (the non-local block reads FLAGS)."""
    mod = types.ModuleType("utils.config")
    mod.FLAGS = types.SimpleNamespace()
    monkeypatch.setitem(sys.modules, "utils.config", mod)
    return mod


def _rel(a, b):
    return float((a - b).norm() / (b.norm() + 1e-30))


def _flat(d, keys):
    return torch.cat([d[k].detach().double().flatten().cpu() for k in keys])


@pytest.mark.parametrize("name", ["mobilenet_v2", "autonl_l"])
def test_three_fused_tail_steps_vs_fp32_reference(built_lib, flags, name):
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
    ts = TrainStep(model, B, image_size=fl["image_size"], fused_tail=True, **kw)
    g = torch.Generator().manual_seed(0)
    keys = [k for k, _ in model.named_parameters()]
    n0 = engine.TRAIN_TAIL_CALLS
    rows = []
    for i in range(3):
        x = torch.randn(B, 3, 224, 224, generator=g).bfloat16()
        t = torch.randint(0, 1000, (B,), generator=g)
        xd, td = x.to(dev).float(), t.to(dev)
        lt = ref32.step(xd, td) - float(tm.l2_loss_mnas(ref32.model, fl["weight_decay"]))
        la = ref16.step(xd.contiguous(memory_format=torch.channels_last), td) - float(
            tm.l2_loss_mnas(ref16.model, fl["weight_decay"]))
        lo = float(ts(x, t))
        rows.append("step %d loss ours %.6f fp32 %.6f autocast %.6f" % (i, lo, lt, la))
        assert abs(lo - lt) <= 2.0 * abs(la - lt) + 5e-3 * abs(lt), rows
    torch.cuda.synchronize()
    assert ts.graph is not None and engine.TRAIN_TAIL_CALLS >= n0 + 3   # 2 eager + the capture
    assert not engine.TRAIN_TAIL_FUSED                                  # scoped to the step
    pt, pa, po = (dict(m.named_parameters()) for m in (ref32.model, ref16.model, model))
    p0f = _flat(p0, keys)
    eo, ea = _rel(_flat(po, keys) - p0f, _flat(pt, keys) - p0f), _rel(_flat(pa, keys) - p0f,
                                                                     _flat(pt, keys) - p0f)
    rows.append("update rel-L2 ours %.4f autocast %.4f" % (eo, ea))
    assert eo <= 1.3 * ea + 1e-2, rows
    bt, ba, bo = (dict(m.named_buffers()) for m in (ref32.model, ref16.model, model))
    for kind in ("running_mean", "running_var"):
        ks = [k for k in bt if k.endswith(kind)]
        e_o = sorted(_rel(bo[k].double().cpu(), bt[k].double().cpu()) for k in ks)
        e_a = sorted(_rel(ba[k].double().cpu(), bt[k].double().cpu()) for k in ks)
        mo, ma = sum(e_o) / len(e_o), sum(e_a) / len(e_a)
        qo, qa = e_o[int(0.9 * (len(e_o) - 1))], e_a[int(0.9 * (len(e_a) - 1))]
        rows.append("%s mean ours %.2e autocast %.2e p90 ours %.2e autocast %.2e"
                    % (kind, mo, ma, qo, qa))
        assert mo <= 1.5 * ma + 2e-3 and qo <= 1.5 * qa + 2e-3, rows


def _small_mbv2(seed):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    from yet_another_mobilenet_series_b200 import mobilenet_supernet as sup
    torch.manual_seed(seed)
    rows = [[1, 16, 1, 1, [3]], [6, 24, 2, 2, [3]], [6, 32, 1, 2, [5]], [6, 64, 1, 2, [3]],
            [6, 96, 1, 2, [3]]]
    model = sup.Model(num_classes=100, input_size=64, inverted_residual_setting=rows,
                      active_fn="nn.ReLU6", batch_norm_momentum=0.01, batch_norm_epsilon=1e-3,
                      last_channel=256)
    model.apply(mb.init_weights_mnas)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    return model.cuda()


def _batch(i, n=16):
    g = torch.Generator().manual_seed(100 + i)
    return (torch.randn(n, 3, 64, 64, generator=g).bfloat16(),
            torch.randint(0, 100, (n,), generator=g))


def _snap(ts, loss):
    out = {"loss": loss.clone()}
    for n, p in ts.model.named_parameters():
        out["p." + n] = p.detach().clone()
        out["ema." + n] = ts.opt.ema_shadow(p).clone()
        for k, v in ts.opt.state.get(p, {}).items():
            out["opt.%s.%s" % (n, k)] = v.clone() if torch.is_tensor(v) else torch.tensor(v)
    for n, b in ts.model.named_buffers():
        out["buf." + n] = b.clone()
    return out


def _same(a, b):
    assert a.keys() == b.keys()
    diff = [k for k in a if not torch.equal(a[k], b[k])]
    assert not diff, diff[:5]


def test_micro_batches_train(built_lib):
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    ts = TrainStep(_small_mbv2(0), 16, image_size=64, micro_batch=4, fused_tail=True)
    n0 = engine.TRAIN_TAIL_CALLS
    losses = [float(ts(*_batch(i % 2))) for i in range(8)]
    assert ts.graph is not None and engine.TRAIN_TAIL_CALLS >= n0 + 4 * 3
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
    # the same step without the flag: close, not the same bits (the pool's order differs)
    ref = TrainStep(_small_mbv2(0), 16, image_size=64, micro_batch=4)
    lr = [float(ref(*_batch(i % 2))) for i in range(8)]
    assert abs(losses[-1] - lr[-1]) <= 0.05 * abs(lr[-1]), (losses, lr)


def test_fused_tail_resume_is_bit_exact(built_lib, tmp_path):
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    ts = TrainStep(_small_mbv2(0), 16, image_size=64, fused_tail=True)
    a = [_snap(ts, ts(*_batch(i))) for i in range(6)]
    assert ts.graph is not None
    ts = TrainStep(_small_mbv2(0), 16, image_size=64, fused_tail=True)
    for i in range(3):
        _same(a[i], _snap(ts, ts(*_batch(i))))     # two fresh runs: the same bits
    path = str(tmp_path / "ckpt.pt")
    ts.save_status(path, 0, 0.0, None)
    ts = TrainStep(_small_mbv2(1), 16, image_size=64, fused_tail=True)
    ts.load_state_dict(torch.load(path, map_location="cpu"))
    for i in range(3, 6):
        _same(a[i], _snap(ts, ts(*_batch(i))))
    assert ts.graph is not None


def test_plain_forward_outside_the_step_is_unchanged(built_lib):
    """TrainStep(fused_tail=True) leaves the switch off: model(x) afterwards launches the unfused
    head, the same bits as a model that never saw the flag."""
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    m = _small_mbv2(0)
    ts = TrainStep(m, 16, image_size=64, fused_tail=True, use_graph=False)
    ts(*_batch(0))
    n0 = engine.TRAIN_TAIL_CALLS
    x = _batch(1)[0].cuda()
    y = m(x)
    assert engine.TRAIN_TAIL_CALLS == n0 and y.shape == (16, 100)
