"""GPU: bit-reproducible Squeeze-and-Excitation and non-local reductions.

1. Every entry point whose CTAs share outputs (yamb_se_pool_fwd, yamb_se_bwd_reduce_bwd,
   yamb_se_fc_fwd, yamb_se_fc_bwd, yamb_nl_gram_fwd), at shapes with several CTAs per output:
   called twice on the same inputs, the second time while an unrelated torch workload runs on
   another stream (a different CTA schedule), the results are the same bits; each is checked
   against fp64 torch.
2. The whole training step of AtomNAS-C+, AutoNL-L and AutoNL-L with `nl_norm: nn.InstanceNorm`:
   the same iteration run eagerly twice and once as a CUDA-graph replay gives the same loss,
   parameters, running statistics and EMA shadows, bit for bit.
3. Two fresh models from the same seed, three TrainStep iterations each (Dropout on, graph
   captured): the same bits.  Two bn_calibration passes (reference utils/common.py:175-187) of
   AutoNL-L from the same state: the same running statistics."""
import gc
import importlib
import sys
import types

import pytest
import torch
import torch.nn.functional as F

from _cfg import MODULE_MAP, load_cfgs

pytestmark = pytest.mark.gpu
ACT_RELU, ACT_SWISH = 1, 3
TOL = 2e-5                       # rel-L2 of an fp32 sum against fp64


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _twice(call):
    """call() -> list of output tensors; run it twice, the second time next to a large matmul
    chain on another stream, and return both results."""
    first = [t.clone() for t in call()]
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    a = torch.randn(4096, 4096, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        for _ in range(8):
            a = torch.tanh(a @ a)
    second = [t.clone() for t in call()]
    torch.cuda.synchronize()
    return first, second


def _launch(fn, st):
    from yet_another_mobilenet_series_b200 import engine
    engine.launch(fn, st)


# ---- 1. entry points -------------------------------------------------------------------------
def _act_bf16(h, scale, shift, act):
    z = h.float() * scale + shift
    z = torch.relu(z) if act == ACT_RELU else z * torch.sigmoid(z)
    return z.bfloat16().double()


@pytest.mark.parametrize("N,HW,C", [(37, 784, 240), (256, 196, 1152), (64, 49, 2560)])
def test_se_pool_and_dgate(built_lib, N, HW, C):
    from yet_another_mobilenet_series_b200 import native as nat
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(N + HW + C)
    h = torch.randn(N * HW, C, generator=g).bfloat16().to(dev)
    dy = torch.randn(N * HW, C, generator=g).bfloat16().to(dev)
    scale = (torch.rand(C, generator=g) + 0.5).to(dev)
    shift = (torch.randn(C, generator=g) * 0.3).to(dev)
    pooled = torch.empty(N, C, device=dev)
    dgate = torch.empty(N, C, device=dev)

    def call():
        p = nat.SePool()
        p.N, p.HW, p.C, p.ldh = N, HW, C, C
        p.h, p.scale, p.shift, p.act = h.data_ptr(), scale.data_ptr(), shift.data_ptr(), ACT_RELU
        p.pooled = pooled.data_ptr()
        _launch(nat.lib().yamb_se_pool_fwd, p)
        r = nat.SeBwdReduce()
        r.N, r.HW, r.C, r.ldd, r.ldh = N, HW, C, C, C
        r.dy, r.h = dy.data_ptr(), h.data_ptr()
        r.scale, r.shift, r.act = scale.data_ptr(), shift.data_ptr(), ACT_RELU
        r.dgate = dgate.data_ptr()
        _launch(nat.lib().yamb_se_bwd_reduce_bwd, r)
        return [pooled, dgate]

    (p1, d1), (p2, d2) = _twice(call)
    assert torch.equal(p1, p2) and torch.equal(d1, d2)
    x = _act_bf16(h, scale, shift, ACT_RELU).view(N, HW, C)
    assert _rel(p1, x.mean(1)) < TOL
    assert _rel(d1, (dy.double().view(N, HW, C) * x).sum(1)) < TOL


@pytest.mark.parametrize("N,C,R", [(33, 480, 20), (100, 1390, 96), (256, 1152, 48),
                                   (256, 2310, 96)])
def test_se_fc_fwd_bwd(built_lib, N, C, R):
    """(C, R) of the SE branches of AutoNL-L (1152, 48) and AtomNAS-C+ (1390 / 2310 hidden
    channels, R = 96): the split-K products have several K slabs, N > 32 several sample slabs."""
    from yet_another_mobilenet_series_b200 import native as nat
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(N * 3 + C + R)
    rnd = lambda *s, sc=1.0: (torch.randn(*s, generator=g) * sc).to(dev)
    pooled = rnd(N, C)
    w_r, b_r = rnd(R, C, sc=C ** -0.5), rnd(R, sc=0.1)
    w_e, b_e = rnd(C, R, sc=R ** -0.5), rnd(C, sc=0.1)
    u, v, gate = (torch.empty(N, R, device=dev), torch.empty(N, R, device=dev),
                  torch.empty(N, C, device=dev))

    def fwd():
        f = nat.SeFc()
        f.N, f.C, f.R, f.act = N, C, R, ACT_SWISH
        f.pooled = pooled.data_ptr()
        f.w_r, f.b_r, f.w_e, f.b_e = w_r.data_ptr(), b_r.data_ptr(), w_e.data_ptr(), b_e.data_ptr()
        f.u, f.v, f.gate = u.data_ptr(), v.data_ptr(), gate.data_ptr()
        _launch(nat.lib().yamb_se_fc_fwd, f)
        return [u, v, gate]

    (u1, v1, g1), second = _twice(fwd)
    assert all(torch.equal(a, b) for a, b in zip((u1, v1, g1), second))
    d = lambda t: t.double().cpu()
    u_ref = d(pooled) @ d(w_r).T + d(b_r)
    v_ref = F.silu(u_ref)
    assert _rel(u1, u_ref) < TOL and _rel(v1, v_ref) < TOL
    assert _rel(g1, torch.sigmoid(d(v1) @ d(w_e).T + d(b_e))) < TOL

    # backward on the saved u / v / gate; the parameter gradients accumulate (+=) onto non-zero
    # values already in the arena
    dgate = rnd(N, C)
    inv_hw = 1.0 / 49
    dpool, dt, du = (torch.empty(N, C, device=dev), torch.empty(N, C, device=dev),
                     torch.empty(N, R, device=dev))
    g0 = {"wr": rnd(R, C), "br": rnd(R), "we": rnd(C, R), "be": rnd(C)}
    grads = {k: t.clone() for k, t in g0.items()}

    def bwd():
        for k in grads:
            grads[k].copy_(g0[k])
        b = nat.SeFcBwd()
        b.N, b.C, b.R, b.act, b.inv_hw = N, C, R, ACT_SWISH, inv_hw
        b.dgate, b.gate, b.u, b.v = dgate.data_ptr(), g1.data_ptr(), u1.data_ptr(), v1.data_ptr()
        b.pooled, b.w_r, b.w_e = pooled.data_ptr(), w_r.data_ptr(), w_e.data_ptr()
        b.dpool, b.dt, b.du = dpool.data_ptr(), dt.data_ptr(), du.data_ptr()
        b.g_wr, b.g_br, b.g_we, b.g_be = (grads[k].data_ptr() for k in ("wr", "br", "we", "be"))
        _launch(nat.lib().yamb_se_fc_bwd, b)
        return [dpool, dt, du] + [grads[k] for k in ("wr", "br", "we", "be")]

    first, second = _twice(bwd)
    assert all(torch.equal(a, b) for a, b in zip(first, second))
    dpool1, dt1, du1, gwr, gbr, gwe, gbe = first
    gt = d(g1)
    dt_ref = d(dgate) * gt * (1 - gt)
    uu = d(u1)
    su = torch.sigmoid(uu)
    du_ref = (dt_ref @ d(w_e)) * (su * (1 + uu * (1 - su)))
    assert _rel(dt1, dt_ref) < TOL and _rel(du1, du_ref) < TOL
    assert _rel(dpool1, (du_ref @ d(w_r)) * inv_hw) < TOL
    assert _rel(gwe, d(g0["we"]) + dt_ref.T @ d(v1)) < TOL
    assert _rel(gbe, d(g0["be"]) + dt_ref.sum(0)) < TOL
    assert _rel(gwr, d(g0["wr"]) + du_ref.T @ d(pooled)) < TOL
    assert _rel(gbr, d(g0["br"]) + du_ref.sum(0)) < TOL


# forward F = phi^T g on the sub-sampled pixels (X = Y = l), and the backward dF = theta^T df over
# every pixel (two tensors)
@pytest.mark.parametrize("N,H,C,I,sub,backward", [(64, 28, 80, 40, 1, False),
                                                  (64, 28, 80, 40, 2, False),
                                                  (64, 28, 80, 40, 1, True),
                                                  (128, 14, 96, 47, 1, True),
                                                  (128, 14, 192, 96, 2, False)])
def test_nl_gram(built_lib, N, H, C, I, sub, backward):
    from yet_another_mobilenet_series_b200 import native as nat
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(N + H + C + I + sub)
    X = torch.randn(N * H * H, C, generator=g).bfloat16().to(dev)
    Y = torch.randn(N * H * H, C, generator=g).bfloat16().to(dev) if backward else X
    G = torch.empty(N, I, C, device=dev)
    alpha = 0.75

    def call():
        a = nat.NlGram()
        a.N, a.H, a.W, a.sub = N, H, H, sub
        a.X, a.ldx, a.I = X.data_ptr(), C, I
        a.Y, a.ldy, a.J = Y.data_ptr(), C, C
        a.alpha, a.G = alpha, G.data_ptr()
        _launch(nat.lib().yamb_nl_gram_fwd, a)
        return [G]

    (g1,), (g2,) = _twice(call)
    assert torch.equal(g1, g2)
    xs = X.double().cpu().view(N, H, H, C)[:, ::sub, ::sub].reshape(N, -1, C)
    ys = Y.double().cpu().view(N, H, H, C)[:, ::sub, ::sub].reshape(N, -1, C)
    assert _rel(g1, alpha * xs[:, :, :I].transpose(1, 2) @ ys) < TOL


# ---- 2. and 3. whole training steps ------------------------------------------------------------
SIZE, B = 128, 64               # reduced input; N = 64 keeps the sample slabs and split-K active
CONFIGS = ["atomnas_c+", "autonl_l", "autonl_l_in"]


@pytest.fixture
def flags(monkeypatch):
    """A stand-in for the reference's utils.config; FLAGS.nl_norm selects the non-local norm."""
    mod = types.ModuleType("utils.config")
    mod.FLAGS = types.SimpleNamespace()
    monkeypatch.setitem(sys.modules, "utils.config", mod)
    return mod


def _build(name, flags, dropout=False):
    """The config's model (tests/golden/model_cfgs.json) at SIZE x SIZE, seeded; the non-local
    norms get gamma = 0.5 (ZeroInitBN would leave the non-local backward all zeros)."""
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    base = name[:-3] if name.endswith("_in") else name
    flags.FLAGS = types.SimpleNamespace(nl_norm="nn.InstanceNorm") if name.endswith("_in") \
        else types.SimpleNamespace()
    cfg = load_cfgs()[base]
    lib = importlib.import_module(MODULE_MAP[cfg["flags"]["model"]])
    torch.manual_seed(cfg["flags"]["random_seed"])
    model = lib.Model(**cfg["model_kwparams"], input_size=SIZE)
    model.apply(mb.init_weights_mnas)
    for m in model.modules():
        if isinstance(m, mb.Nonlocal):
            m.bn.weight.data.fill_(0.5)
        if isinstance(m, torch.nn.Dropout) and not dropout:
            m.p = 0.0
    if name.endswith("_in"):
        assert any(isinstance(m, torch.nn.InstanceNorm2d) for m in model.modules())
    return model.cuda()


def _batch(seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, 3, SIZE, SIZE, generator=g).to(torch.bfloat16),
            torch.randint(0, 1000, (B,), generator=g))


def _snapshot(ts, model):
    A = ts.opt.arenas()
    out = {k: A[k].clone() for k in ("p", "ema") if A.get(k) is not None}
    out.update({"buf." + k: v.clone() for k, v in model.named_buffers()})
    out.update({"shadow.%d" % i: s.clone() for i, s in enumerate(ts.stat_shadow)})
    return out


def _restore(ts, model, st):
    A = ts.opt.arenas()
    with torch.no_grad():
        for k in ("p", "sq", "mom", "ema", "bf16"):
            if k in st:
                A[k].copy_(st[k])
        for k, v in model.named_buffers():
            v.copy_(st["buf"][k])
        for s, v in zip(ts.stat_shadow, st["shadow"]):
            s.copy_(v)
    ts.global_step = st["step"]


def _diff(a, b):
    assert a.keys() == b.keys()
    return [k for k in a if not torch.equal(a[k], b[k])]


@pytest.mark.parametrize("name", CONFIGS)
def test_graph_replay_equals_eager(built_lib, flags, name):
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    model = _build(name, flags)
    kinds = {type(m).__name__ for m in model.modules()}
    assert "SqueezeAndExcitation" in kinds
    assert ("Nonlocal" in kinds) == (name != "atomnas_c+")
    x, t = _batch(0)
    ts = TrainStep(model, B, image_size=SIZE)
    for _ in range(2):
        ts(x, t)                                  # two eager warm-up iterations
    torch.cuda.synchronize()
    A = ts.opt.arenas()
    st = {k: A[k].clone() for k in ("p", "sq", "mom", "ema", "bf16") if A.get(k) is not None}
    st["buf"] = {k: v.clone() for k, v in model.named_buffers()}
    st["shadow"] = [s.clone() for s in ts.stat_shadow]
    st["step"] = ts.global_step
    ts.use_graph = False
    loss_e = ts(x, t).clone()
    snap_e = _snapshot(ts, model)
    _restore(ts, model, st)
    loss_e2 = ts(x, t).clone()
    snap_e2 = _snapshot(ts, model)
    _restore(ts, model, st)
    ts.use_graph = True
    loss_g = ts(x, t).clone()                     # captures, then replays
    torch.cuda.synchronize()
    assert ts.graph is not None
    snap_g = _snapshot(ts, model)
    assert torch.equal(loss_e, loss_e2) and torch.equal(loss_e, loss_g), (loss_e, loss_e2, loss_g)
    assert not _diff(snap_e, snap_e2), _diff(snap_e, snap_e2)[:5]
    assert not _diff(snap_e, snap_g), _diff(snap_e, snap_g)[:5]


def _three_steps(name, flags):
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    model = _build(name, flags, dropout=True)
    assert any(isinstance(m, torch.nn.Dropout) and m.p > 0 for m in model.modules())
    ts = TrainStep(model, B, image_size=SIZE)
    losses = [ts(*_batch(i)).clone() for i in range(3)]
    torch.cuda.synchronize()
    assert ts.graph is not None                   # the third call replayed the graph
    out = _snapshot(ts, model)
    out.update({"loss.%d" % i: l for i, l in enumerate(losses)})
    del ts, model
    gc.collect()
    return out


@pytest.mark.parametrize("name", CONFIGS)
def test_run_to_run(built_lib, flags, name):
    a = _three_steps(name, flags)
    b = _three_steps(name, flags)
    assert not _diff(a, b), _diff(a, b)[:5]


def test_bn_calibration_run_to_run(built_lib, flags):
    """Two bn_calibration passes of AutoNL-L from the same state: model in eval mode, every
    BatchNorm reset, in train mode with cumulative statistics (momentum None), two batches."""
    model = _build("autonl_l", flags)
    state = {k: v.clone() for k, v in model.state_dict().items()}

    def bn_calibration(m):
        if isinstance(m, torch.nn.BatchNorm2d):
            m.reset_running_stats()
            m.train()
            m.momentum = None

    runs = []
    for _ in range(2):
        model.load_state_dict(state)
        model.eval()
        model.apply(bn_calibration)
        with torch.no_grad():
            for i in range(2):
                model(_batch(10 + i)[0].cuda())
        torch.cuda.synchronize()
        runs.append({k: v.clone() for k, v in model.named_buffers() if "running_" in k})
    assert not _diff(runs[0], runs[1]), _diff(runs[0], runs[1])[:5]
    assert any(float(v.abs().sum()) > 0 for k, v in runs[0].items() if "running_mean" in k)
