"""GPU: the eval-mode stem (yamb_stem_conv_eval_fwd) and head + pool (yamb_head_pool_eval_fwd)
kernels and their opt-in dispatch (engine.EVAL_TAIL_FUSED).

- stem: bitwise equal to the stem kernel -> eval_coeffs -> bn_apply sequence, every Cout / act;
- head: every pooled element within 2 bf16 ulps of the fp64 mean of the unfused path's a,
  rounded to bf16; HW 1 / 49 / 64 / 100, the heads of all four configurations and two more
  widths;
- both kernels: the same bits on two runs; an uncovered shape returns YAMB_EINVAL and the
  dispatcher falls back;
- switch off: a MobileNetV2 eval forward launches the unfused sequence and computes its bits."""
import ctypes as C

import pytest
import torch

from _cfg import build_from_cfg

pytestmark = pytest.mark.gpu
ACTS = ["nn.Identity", "nn.ReLU", "nn.ReLU6", "nn.Swish", "nn.HSwish"]
_X = {}


def _act(name):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    if name == "nn.Identity":
        return mb.Identity
    return mb.get_active_fn(name)


def _randomise_bn(bn, g):
    with torch.no_grad():
        bn.weight.copy_(torch.rand(bn.num_features, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(bn.num_features, generator=g) * 0.3)
        bn.running_mean.copy_(torch.randn(bn.num_features, generator=g) * 0.3)
        bn.running_var.copy_(torch.rand(bn.num_features, generator=g) + 0.5)


def _image(N, H, W):
    if (N, H, W) not in _X:
        g = torch.Generator().manual_seed(N * 7 + H + W)
        _X[(N, H, W)] = torch.randn(N, 3, H, W, generator=g).bfloat16().cuda().contiguous(
            memory_format=torch.channels_last)
    return _X[(N, H, W)]


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("cout", [8, 16, 32, 64])
def test_stem_eval_bitwise(built_lib, monkeypatch, cout, act):
    from yet_another_mobilenet_series_b200 import engine, tail_ops
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    g = torch.Generator().manual_seed(cout)
    mod = mb.ConvBNReLU(3, cout, stride=2, active_fn=_act(act))
    _randomise_bn(mod[1], g)
    mod = mod.cuda().eval()
    for N, H, W in ((1, 224, 224), (3, 224, 224), (256, 224, 224), (1, 113, 97), (3, 113, 97),
                    (256, 113, 97)):
        x = _image(N, H, W)
        with torch.no_grad():
            monkeypatch.setattr(engine, "EVAL_TAIL_FUSED", False)
            c0, l0 = engine.EVAL_TAIL_CALLS, engine.LAUNCHES
            old = mod(x)
            assert engine.EVAL_TAIL_CALLS == c0 and engine.LAUNCHES == l0 + 2
            monkeypatch.setattr(engine, "EVAL_TAIL_FUSED", True)
            new = mod(x)
            again = mod(x)
            assert engine.EVAL_TAIL_CALLS == c0 + 2 and engine.LAUNCHES == l0 + 4
        torch.cuda.synchronize()
        assert new.shape == old.shape and new.is_contiguous(memory_format=torch.channels_last)
        assert torch.equal(new, old), (N, H, W, (new.float() - old.float()).abs().max())
        assert torch.equal(new, again)


def _ulp_bf16(v):
    """bf16 unit in the last place of |v| (fp64), at least the smallest normal's."""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


HEAD_SHAPES = [(320, 1280, "nn.ReLU"), (320, 1280, "nn.ReLU6"), (320, 1280, "nn.Swish"),
               (64, 200, "nn.HSwish"), (512, 136, "nn.Identity")]


@pytest.mark.parametrize("cin,cout,act", HEAD_SHAPES)
@pytest.mark.parametrize("hw", [1, 49, 64, 100])
def test_head_pool_eval(built_lib, monkeypatch, cin, cout, act, hw):
    from yet_another_mobilenet_series_b200 import engine, tail_ops
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    side = {1: (1, 1), 49: (7, 7), 64: (8, 8), 100: (10, 10)}[hw]
    g = torch.Generator().manual_seed(cin + cout + hw)
    mod = mb.ConvBNReLU(cin, cout, kernel_size=1, active_fn=_act(act))
    mod.apply(mb.init_weights_mnas)
    _randomise_bn(mod[1], g)
    mod = mod.cuda().eval()
    for N in (1, 5, 256):
        x = torch.randn(N, cin, *side, generator=g).bfloat16().cuda().contiguous(
            memory_format=torch.channels_last)
        with torch.no_grad():
            monkeypatch.setattr(engine, "EVAL_TAIL_FUSED", False)
            assert tail_ops.head_pool_eval(mod, x) is None        # switch off: not taken
            a = tail_ops.pw_conv_bn_act(mod, x)                    # the unfused path's a
            monkeypatch.setattr(engine, "EVAL_TAIL_FUSED", True)
            c0 = engine.EVAL_TAIL_CALLS
            p1 = tail_ops.head_pool_eval(mod, x)
            p2 = tail_ops.head_pool_eval(mod, x)
            assert engine.EVAL_TAIL_CALLS == c0 + 2
        torch.cuda.synchronize()
        assert p1.shape == (N, cout, 1, 1) and p1.dtype == torch.bfloat16
        want = a.double().mean((2, 3)).bfloat16().double()
        got = p1.view(N, cout).double()
        err = (got - want).abs() / _ulp_bf16(want)
        assert float(err.max()) <= 2.0, (N, float(err.max()))
        assert torch.equal(p1, p2)


def test_uncovered_shapes_fall_back(built_lib, monkeypatch):
    from yet_another_mobilenet_series_b200 import engine, tail_ops
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    from yet_another_mobilenet_series_b200 import native as nat
    lib = nat.lib()
    dev = torch.device("cuda")
    # the kernels themselves: Cin > 512 (head), Cout = 72 (stem) -> YAMB_EINVAL, nothing enqueued
    x = torch.zeros(2, 4, 520, device=dev, dtype=torch.bfloat16)
    w = torch.zeros(64, 520, device=dev, dtype=torch.bfloat16)
    f = torch.zeros(64, device=dev)
    out = torch.zeros(2, 64, device=dev, dtype=torch.bfloat16)
    a = nat.HeadPoolEval()
    a.N, a.HW, a.Cin, a.Cout = 2, 4, 520, 64
    a.x, a.w, a.scale, a.shift, a.pooled = x.data_ptr(), w.data_ptr(), f.data_ptr(), \
        f.data_ptr(), out.data_ptr()
    assert lib.yamb_head_pool_eval_fwd(C.byref(a), nat.stream_handle()) == nat.EINVAL
    s = nat.StemConvEval()
    xi = torch.zeros(1, 8, 8, 3, device=dev, dtype=torch.bfloat16)
    wi = torch.zeros(72, 27, device=dev)
    yi = torch.zeros(1, 4, 4, 72, device=dev, dtype=torch.bfloat16)
    f72 = torch.zeros(72, device=dev)
    s.conv.N, s.conv.H, s.conv.W, s.conv.Cout = 1, 8, 8, 72
    s.conv.x, s.conv.w, s.conv.y = xi.data_ptr(), wi.data_ptr(), yi.data_ptr()
    s.scale, s.shift = f72.data_ptr(), f72.data_ptr()
    assert lib.yamb_stem_conv_eval_fwd(C.byref(s), nat.stream_handle()) == nat.EINVAL
    # the dispatcher: a 520-channel head falls back to the unfused sequence with the same bits
    mod = mb.ConvBNReLU(520, 64, kernel_size=1, active_fn=mb.get_active_fn("nn.ReLU"))
    _randomise_bn(mod[1], torch.Generator().manual_seed(5))
    mod = mod.cuda().eval()
    xh = torch.randn(3, 520, 7, 7).bfloat16().cuda().contiguous(memory_format=torch.channels_last)
    with torch.no_grad():
        monkeypatch.setattr(engine, "EVAL_TAIL_FUSED", True)
        c0 = engine.EVAL_TAIL_CALLS
        assert tail_ops.head_pool_eval(mod, xh) is None
        assert engine.EVAL_TAIL_CALLS == c0
        # a gradient wanted, or a BatchNorm on batch statistics: not taken either
    mod2 = mb.ConvBNReLU(320, 64, kernel_size=1, active_fn=mb.get_active_fn("nn.ReLU")).cuda()
    x2 = torch.randn(3, 320, 7, 7).bfloat16().cuda().contiguous(memory_format=torch.channels_last)
    mod2.eval()
    assert tail_ops.head_pool_eval(mod2, x2) is None                       # grad enabled
    with torch.no_grad():
        mod2.train()
        assert tail_ops.head_pool_eval(mod2, x2) is None                   # batch statistics
        mod2.eval()
        assert tail_ops.head_pool_eval(mod2, x2) is not None
    assert engine.EVAL_TAIL_CALLS == c0 + 1


def test_switch_off_keeps_the_eval_forward(built_lib, monkeypatch):
    """MobileNetV2 eval forward with the switch off: the unfused stem and head sequences (two
    launches each, torch's mean for the pool), the same logits as those layers run one by one;
    with the switch on: two launches fewer."""
    from yet_another_mobilenet_series_b200 import engine, tail_ops
    from yet_another_mobilenet_series_b200 import mobilenet_supernet as sup
    model, _ = build_from_cfg("mobilenet_v2", seed=3)
    model = model.cuda().eval()
    x = _image(4, 224, 224)
    monkeypatch.setattr(engine, "EVAL_TAIL_FUSED", False)
    with torch.no_grad():
        c0, l0 = engine.EVAL_TAIL_CALLS, engine.LAUNCHES
        y_off = model(x)
        n_off = engine.LAUNCHES - l0
        assert engine.EVAL_TAIL_CALLS == c0
        # the same layers by hand: stem kernel + bn_apply, blocks, head GEMM + bn_apply, mean, fc
        h = x
        feats = list(model.features)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            h = tail_ops.stem_conv_bn_act(feats[0], h)
            for blk in feats[1:-2]:
                h = blk(h)
            h = tail_ops.pw_conv_bn_act(feats[-2], h)
            h = h.mean((2, 3), keepdim=True).flatten(1)
            y_hand = sup.run_classifier(model.classifier, h).float()
        monkeypatch.setattr(engine, "EVAL_TAIL_FUSED", True)
        l1 = engine.LAUNCHES
        y_on = model(x)
        n_on = engine.LAUNCHES - l1
        assert engine.EVAL_TAIL_CALLS == c0 + 2
    torch.cuda.synchronize()
    assert torch.equal(y_off, y_hand)
    assert n_on == n_off - 2, (n_on, n_off)
    rel = float((y_on - y_off).norm() / y_off.norm())
    assert rel < 1e-2, rel
