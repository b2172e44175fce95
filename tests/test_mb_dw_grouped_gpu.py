"""GPU: the depthwise of every branch of a multi-branch training block in one launch each way
(TrainStep(grouped_branches=True), engine.TRAIN_MB_DW_GROUPED) against the per-branch launches,
bit for bit: real AtomNAS-C and C+ blocks (k in {3, 5, 7}, stride 1 and 2, odd widths through the
padded shadow) and a [3, 5, 7] supernet block, then whole TrainStep steps."""
import ctypes as C
import copy
import os
import sys
import types

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_cfg(name):
    """Model and config of an AtomNAS configuration (tests/golden/model_cfgs_multi_branch.json)."""
    import importlib
    import json
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    from yet_another_mobilenet_series_b200 import searched_network  # noqa: F401
    with open(os.path.join(ROOT, "tests", "golden", "model_cfgs_multi_branch.json")) as f:
        cfg = json.load(f)[name]
    lib = importlib.import_module(cfg["flags"]["model"].replace(
        "models.", "yet_another_mobilenet_series_b200."))
    torch.manual_seed(0)
    model = lib.Model(**cfg["model_kwparams"], input_size=cfg["flags"]["image_size"])
    model.apply(mb.init_weights_mnas)
    return model, cfg


@pytest.fixture(autouse=True)
def every_kind(monkeypatch):
    """Every multi-branch block takes the grouped path (the shape rule off)."""
    from yet_another_mobilenet_series_b200 import engine
    monkeypatch.setattr(engine, "MB_DW_SHAPE_RULE", False)


@pytest.fixture
def flags(monkeypatch):
    mod = types.ModuleType("utils.config")
    mod.FLAGS = types.SimpleNamespace()
    monkeypatch.setitem(sys.modules, "utils.config", mod)
    return mod


def _blocks(name):
    """(input H, block) of the multi-branch blocks of `name`, on the GPU."""
    from yet_another_mobilenet_series_b200 import engine
    model, cfg = build_cfg(name)
    out, H = [], cfg["flags"]["image_size"]
    for m in model.features:
        if hasattr(m, "expand_conv") or hasattr(m, "ops"):
            if len(engine.block_parts(m).dws) > 1:
                out.append((H, m))
            H = (H - 1) // m.stride + 1
        else:
            for conv in [c for c in m.modules() if isinstance(c, torch.nn.Conv2d)][:1]:
                H = (H - 1) // conv.stride[0] + 1
    return out


def _pick(blocks):
    """A stride-1 and a stride-2 block, and one with a width that is not a multiple of 8, each
    kind once."""
    seen, out = set(), []
    for H, m in blocks:
        odd = any(c % 8 for c in m.channels)
        key = (m.stride, odd, H)
        if key not in seen and (m.stride == 2 or odd or len(out) < 2):
            seen.add(key)
            out.append((H, m))
    return out[:6]


def _run(block, x, dy, grouped, prof=None):
    from yet_another_mobilenet_series_b200 import engine
    engine.TRAIN_MB_DW_GROUPED = grouped
    engine.PROFILE = prof
    try:
        xg = x.clone().requires_grad_(True)
        y = block(xg)
        y.backward(dy)
        torch.cuda.synchronize()
    finally:
        engine.TRAIN_MB_DW_GROUPED = False
        engine.PROFILE = None
    out = {"y": y.detach().clone(), "dx": xg.grad.clone()}
    for n, p in block.named_parameters():
        out["g." + n] = p.grad.clone()
    for n, b in block.named_buffers():
        out["b." + n] = b.clone()
    return out


def _same(a, b):
    assert a.keys() == b.keys()
    diff = [k for k in a if not torch.equal(a[k], b[k])]
    assert not diff, diff[:8]


def _block_parity(H, m, N=32):
    from yet_another_mobilenet_series_b200 import engine
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(11)
    Ho = (H - 1) // m.stride + 1
    x = torch.randn(N, m.input_dim, H, H, generator=g).to(dev)
    dy = torch.randn(N, m.output_dim, Ho, Ho, generator=g).to(dev).bfloat16()
    a, b = copy.deepcopy(m).to(dev).train(), copy.deepcopy(m).to(dev).train()
    ref = _run(a, x, dy, False)
    n0 = engine.TRAIN_MB_DW_GROUPED_CALLS
    prof = []
    got = _run(b, x, dy, True, prof)
    assert engine.TRAIN_MB_DW_GROUPED_CALLS == n0 + 2
    tags = [t[0] for t in prof]
    assert tags.count("dw_fwd_grouped") == 1 and tags.count("dw_bwd_grouped") == 1, tags
    assert not [t for t in tags if t in ("dw_fwd", "dw_bwd")], tags
    _same(ref, got)
    # a second step from the updated running statistics, again bit for bit
    _same(_run(a, x, dy, False), _run(b, x, dy, True))


@pytest.mark.parametrize("name", ["atomnas_c", "atomnas_c+"])
def test_block_parity_atomnas(built_lib, flags, name):
    blocks = _pick(_blocks(name))
    assert any(m.stride == 2 for _, m in blocks)
    ks = set()
    for H, m in blocks:
        ks |= set(m.kernel_sizes)
        _block_parity(H, m)
    assert ks == {3, 5, 7}
    if name == "atomnas_c+":
        assert any(any(c % 8 for c in m.channels) for _, m in blocks)


@pytest.mark.parametrize("stride", [1, 2])
def test_block_parity_supernet(built_lib, stride):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    bn = {"momentum": 0.01, "eps": 1e-3}
    torch.manual_seed(5)
    blk = mb.InvertedResidualChannels(32, 32 if stride == 1 else 40, stride, [96, 96, 96],
                                      [3, 5, 7], True, mb.get_active_fn("nn.ReLU6"), bn)
    blk.apply(mb.init_weights_mnas)
    _block_parity(28, blk)


def test_grids_match_per_branch_launches(built_lib):
    """The grids the grouped launch validates are those of the per-branch launches' sizing, and a
    descriptor with another grid is refused with nothing enqueued."""
    from yet_another_mobilenet_series_b200 import native as nat
    lib = built_lib
    dev = torch.device("cuda", 0)
    N, H, C_ = 4, 56, 48
    t = [torch.zeros(N * H * H, 3 * C_, device=dev, dtype=torch.bfloat16) for _ in range(2)]
    w = [torch.zeros(C_, k * k, device=dev) for k in (3, 5, 7)]
    a = nat.DwBwdGrouped()
    a.nbranch = 3
    for b, k in enumerate((3, 5, 7)):
        d = a.branch[b]
        d.N, d.H, d.W, d.C, d.ldc, d.k, d.stride = N, H, H, C_ if b else 8, 3 * C_, k, 1
        d.dz = d.h = d.x = d.dx = t[0].data_ptr() + 2 * C_ * b
        d.ca = d.cb = d.cc = w[0].data_ptr()
        d.w = d.dw = w[b].data_ptr()
    assert lib.yamb_depthwise_grouped_grids(None, C.byref(a)) == 0
    assert all(a.grid[b] > 0 for b in range(3))
    assert a.grid_wgrad[0] == a.grid_wgrad[1] == 0 and a.grid_wgrad[2] > 0
    for b in range(3):
        one = nat.DwBwdGrouped()
        one.nbranch = 1
        one.branch[0] = a.branch[b]
        assert lib.yamb_depthwise_grouped_grids(None, C.byref(one)) == 0
        assert (one.grid[0], one.grid_wgrad[0]) == (a.grid[b], a.grid_wgrad[b])
    a.grid[1] += 1
    assert lib.yamb_depthwise_bwd_grouped(C.byref(a), nat.stream_handle()) == -1


def _snap(ts, loss):
    out = {"loss": loss.clone(), "top1": ts.top1.clone(), "top5": ts.top5.clone()}
    for n, p in ts.model.named_parameters():
        out["p." + n] = p.detach().clone()
    for n, b in ts.model.named_buffers():
        out["buf." + n] = b.clone()
    for i, s in enumerate(ts.stat_shadow):
        out["stat_ema.%d" % i] = s.clone()
    ema = getattr(ts.opt, "ema_flat", None) or getattr(ts.opt, "ema", None)
    if isinstance(ema, torch.Tensor):
        out["ema"] = ema.clone()
    return out


def _steps(name, steps=3, B=8, **kw):
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    model, cfg = build_cfg(name)
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


@pytest.mark.parametrize("name", ["atomnas_c+", "atomnas_c"])
def test_train_step_bitwise(built_lib, flags, name):
    """Three graph-replayed steps with grouped_branches=True have the default step's bits."""
    from yet_another_mobilenet_series_b200 import engine
    n0 = engine.TRAIN_MB_DW_GROUPED_CALLS
    got = _steps(name, grouped_branches=True)
    assert engine.TRAIN_MB_DW_GROUPED_CALLS > n0
    ref = _steps(name)
    for a, b in zip(ref, got):
        _same(a, b)
    assert not engine.TRAIN_MB_DW_GROUPED


def test_fused_se_fallback_and_combined_switches(built_lib, flags):
    """With fused_se the SE blocks' backward keeps the per-branch depthwise_bwd_se launches: the
    step equals fused_se without grouping bitwise.  Micro-batches and a partial last batch run too."""
    ref = _steps("atomnas_c+", steps=2, fused_se=True, use_graph=False)
    got = _steps("atomnas_c+", steps=2, fused_se=True, grouped_branches=True, use_graph=False)
    for a, b in zip(ref, got):
        _same(a, b)
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    model, cfg = build_cfg("atomnas_c+")
    hw = cfg["flags"]["image_size"]
    ts = TrainStep(model.cuda(), 8, image_size=hw, grouped_branches=True, fused_stem=True,
                   fused_tail=True, fused_expand_dw=True, micro_batch=4, use_graph=False)
    g = torch.Generator().manual_seed(3)
    for n in (8, 5):
        x = torch.randn(n, 3, hw, hw, generator=g).bfloat16()
        t = torch.randint(0, 1000, (n,), generator=g)
        c0 = engine.TRAIN_MB_DW_GROUPED_CALLS
        loss = float(ts(x, t))
        torch.cuda.synchronize()
        assert loss == loss and 0.5 < loss < 20.0
        assert engine.TRAIN_MB_DW_GROUPED_CALLS > c0
    assert not engine.TRAIN_MB_DW_GROUPED
