"""GPU parity of the ONE-LAUNCH eval-mode block (csrc/block_eval.cu, yamb_block_eval_fwd).

Reference semantics: InvertedResidualChannels.forward in model.eval() (reference
models/mobilenet_base.py:446-451 with every BatchNorm on running statistics; validation path
common.py:67-80 under torch.no_grad()).  Checked against

  * the oracle with the kernel's rounding points (oracle.ir_block.forward(..., quant="fused")):
    tight, 3e-3 rel-L2 (bf16 output rounding alone is 1.65e-3, SURVEY.md §8c);
  * the reference's stock-torch graph in fp32 on the same GPU (truth) with the same graph under
    autocast-bf16 as the yardstick: err(ours) <= 1.5 * err(autocast) + 2.5e-3;
  * the four-launch eval sequence of this repo (the path it replaces).

Edge cases: images that do not divide into tiles, odd image counts on the two-images-per-tile
geometry, channel counts that need K / N padding (24), a partial last 64-channel slice (144),
the 320-column project accumulator, three K panels (Cin = 160), stride 2 (incl. odd sizes and a
single output pixel), blocks without the expansion (one and two channel panels, with stride 2).
"""
import copy
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

SLACK, FLOOR = 1.5, 2.5e-3


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _make_block(cin, chid, cout, act, seed, stride=1, expand=True, k=3):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    torch.manual_seed(seed)
    blk = mb.InvertedResidualChannels(cin, cout, stride, [chid], [k], expand,
                                      active_fn=mb.get_active_fn({"relu": "nn.ReLU", "relu6": "nn.ReLU6",
                                                                "swish": "nn.Swish"}[act]),
                                      batch_norm_kwargs={"momentum": 0.01, "eps": 1e-3})
    g = torch.Generator().manual_seed(seed)
    for m in blk.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.weight.data.uniform_(0.5, 1.5, generator=g)
            m.bias.data.normal_(0, 0.3, generator=g)
            m.running_mean.normal_(0, 0.5, generator=g)
            m.running_var.uniform_(0.5, 2.0, generator=g)
        elif isinstance(m, torch.nn.Conv2d):
            m.weight.data.normal_(0, (2.0 / max(1, m.weight[0].numel())) ** 0.5, generator=g)
    return blk.eval()


# (cin, chid, cout, N, H, W, act)
CASES = [
    (24, 144, 24, 4, 56, 56, "relu"),      # MobileNetV2 block 3: K pad, N pad, partial slice
    (32, 192, 32, 4, 28, 28, "relu6"),     # 7x16 tiles, as many as two 7x7 images
    (64, 384, 64, 6, 14, 14, "relu"),
    (64, 384, 96, 5, 14, 14, "relu"),      # block 11: no skip connection
    (96, 576, 96, 3, 14, 14, "relu6"),
    (160, 960, 160, 5, 7, 7, "relu"),      # two images per tile, odd image count, 3 K panels
    (160, 960, 320, 4, 7, 7, "relu"),      # block 17: 320-column accumulator in two halves
    (16, 64, 16, 2, 20, 20, "relu"),       # one slice, tiles overhang the image
    (40, 120, 40, 3, 9, 13, "swish"),      # odd sizes, swish
    (8, 8, 8, 1, 3, 3, "relu"),            # smallest legal block
    (32, 192, 32, 2, 112, 112, "relu"),    # many tiles per CTA
    # stride 2 (7x7 outputs from a 15x15 input tile, 2 channels per stencil thread)
    (16, 96, 24, 2, 112, 112, "relu", 2, True),     # MobileNetV2 block 2
    (24, 144, 32, 3, 56, 56, "relu6", 2, True),     # block 4
    (32, 192, 64, 5, 28, 28, "relu", 2, True),      # block 7
    (96, 576, 160, 3, 14, 14, "relu", 2, True),     # block 14
    (16, 48, 24, 2, 17, 23, "swish", 2, True),      # odd sizes: Ho = 9, Wo = 12
    (8, 16, 8, 1, 2, 2, "relu", 2, True),           # one output pixel
    # no expansion (hidden == input): the stencil reads the x tile itself
    (32, 32, 16, 2, 112, 112, "relu", 1, False),    # MobileNetV2 block 1
    (96, 96, 96, 3, 14, 14, "relu6", 1, False),     # two 64-channel panels, skip connection
    (24, 24, 40, 2, 30, 30, "relu", 2, False),      # no expansion + stride 2
    # 5x5 / 7x7 depthwise (Proxyless-mobile, apps/mobilenet/proxyless_mobile_mnas.yml)
    (16, 48, 32, 2, 112, 112, "relu6", 2, True, 5),   # 112 -> 56, k5 s2: 6x7 outputs per tile
    (40, 120, 40, 3, 28, 28, "relu6", 1, True, 5),    # k5 s1, 7x16 tiles
    (80, 240, 80, 3, 14, 14, "relu6", 1, True, 5),
    (96, 288, 96, 5, 7, 7, "relu", 1, True, 5),       # two images per tile, 5x5
    (32, 96, 40, 2, 56, 56, "relu6", 2, True, 7),     # k7 s2: 4x7 outputs from a 13x19 tile
    (96, 576, 192, 3, 14, 14, "relu6", 2, True, 7),
    (192, 576, 192, 3, 7, 7, "relu6", 1, True, 7),    # k7 s1: one 7x7 image per tile, 3 K panels
    (192, 1152, 320, 2, 7, 7, "relu6", 1, True, 7),   # 18 slices, 320-column accumulator
    (24, 72, 24, 2, 19, 11, "relu", 1, True, 7),      # odd sizes, 7x7
    (24, 72, 24, 2, 19, 11, "relu", 2, True, 5),      # odd sizes, 5x5 stride 2
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "x".join(str(v) for v in c))
def test_fused_eval_block(built_lib, case):
    from oracle import ir_block as ob
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200 import engine
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cin, chid, cout, N, H, W, act = case[:7]
    stride, expand = (case[7], case[8]) if len(case) > 7 else (1, True)
    k = case[9] if len(case) > 9 else 3
    dev = torch.device("cuda")
    blk = _make_block(cin, chid, cout, act, sum(case[:6]), stride, expand, k)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(N, cin, H, W, generator=g).bfloat16().float()
    # ---- oracle with the kernel's rounding points (CPU) ----
    cfg, P = ob.extract(blk)
    yo, _ = ob.forward(x, cfg, P, training=False, quant="fused")
    # ---- this repo: one launch ----
    blk_d = copy.deepcopy(blk).to(dev).eval()
    calls0 = engine.EVAL_FUSED_CALLS
    launches0 = engine.LAUNCHES
    with torch.no_grad():
        y = blk_d(x.to(dev))
    torch.cuda.synchronize()
    assert engine.EVAL_FUSED_CALLS == calls0 + 1, "the block did not take the one-launch path"
    assert engine.LAUNCHES == launches0 + 1
    assert y.shape == yo.shape and y.dtype == torch.bfloat16
    assert torch.isfinite(y.float()).all()
    e_oracle = _rel(y, yo)
    # ---- the four-launch sequence it replaces ----
    engine.EVAL_FUSED = False
    try:
        with torch.no_grad():
            y4 = blk_d(x.to(dev))
        torch.cuda.synchronize()
    finally:
        engine.EVAL_FUSED = True
    assert engine.LAUNCHES - launches0 >= (5 if expand else 4)
    # ---- stock torch fp32 (truth) and autocast-bf16 (yardstick) on the same GPU ----
    ref = tm.as_reference(copy.deepcopy(blk)).to(dev).eval()
    with torch.no_grad():
        yt = ref(x.to(dev))
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ya = ref(x.to(dev).contiguous(memory_format=torch.channels_last))
    eo, ea, e4 = _rel(y, yt), _rel(ya, yt), _rel(y4, yt)
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "block_eval_parity.txt"), "a") as f:
        f.write("%-34s vs oracle(fused points) %.3e | vs fp32: one-launch %.3e  four-launch %.3e  "
                "autocast %.3e\n" % ("x".join(str(v) for v in case), e_oracle, eo, e4, ea))
    assert e_oracle < 3e-3, e_oracle
    assert eo <= SLACK * ea + FLOOR, (eo, ea)
    assert _rel(y, y4) < 1e-2


def test_proxyless_eval_uses_the_one_launch_blocks(built_lib):
    """Proxyless-mobile (k in {3,5,7}, reference apps/mobilenet/proxyless_mobile_mnas.yml): all 20
    blocks in one launch each; logits vs the reference graph in fp32 with the autocast yardstick."""
    from _cfg import build_from_cfg
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200 import engine
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda")
    model, _ = build_from_cfg("proxyless_mobile")
    g = torch.Generator().manual_seed(5)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1, generator=g)
            m.running_var.uniform_(0.8, 1.25, generator=g)
    model = model.to(dev).eval()
    x = torch.randn(8, 3, 224, 224, generator=g).to(dev)
    c0 = engine.EVAL_FUSED_CALLS
    with torch.no_grad():
        y = model(x).float()
    torch.cuda.synchronize()
    assert engine.EVAL_FUSED_CALLS - c0 == 20
    ref = tm.as_reference(copy.deepcopy(model)).eval()
    with torch.no_grad():
        yt = ref(x)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ya = ref(x.contiguous(memory_format=torch.channels_last)).float()
    eo, ea = _rel(y, yt), _rel(ya, yt)
    assert eo <= SLACK * ea + FLOOR, (eo, ea)


def test_fused_eval_needs_no_grad_and_eval_mode(built_lib):
    """Gradient wanted or a BatchNorm in training mode -> the four-launch autograd path."""
    from yet_another_mobilenet_series_b200 import engine
    dev = torch.device("cuda")
    blk = _make_block(32, 192, 32, "relu", 3).to(dev)
    x = torch.randn(2, 32, 14, 14, device=dev)
    c0 = engine.EVAL_FUSED_CALLS
    y = blk(x.clone().requires_grad_(True))           # grad enabled
    assert engine.EVAL_FUSED_CALLS == c0 and y.requires_grad
    blk.train()
    with torch.no_grad():
        blk(x)
    assert engine.EVAL_FUSED_CALLS == c0
    blk.eval()
    with torch.no_grad():
        blk(x)
    assert engine.EVAL_FUSED_CALLS == c0 + 1


def test_fused_eval_abi_rejects_what_it_does_not_cover(built_lib):
    import ctypes as C
    from yet_another_mobilenet_series_b200 import native as nat
    lib = built_lib
    dev = torch.device("cuda")
    buf = torch.zeros(1 << 16, device=dev, dtype=torch.float32)
    a = nat.BlockEval()
    a.N, a.H, a.W, a.Cin, a.Chid, a.Cout = 1, 8, 8, 16, 32, 16
    a.kernel, a.stride, a.act, a.residual = 3, 1, 1, 1
    for f in ("x", "y", "w_expand", "w_dw", "w_project"):
        setattr(a, f, buf.data_ptr())
    for bn in (a.bn1, a.bn2, a.bn3):
        bn.running_mean = bn.running_var = buf.data_ptr()
        bn.eps = 1e-3
    st = torch.cuda.current_stream().cuda_stream
    assert lib.yamb_block_eval_fwd(C.byref(a), st) == 0
    torch.cuda.synchronize()
    for field, bad in (("stride", 3), ("kernel", 4), ("Cin", 12), ("Cout", 328), ("Cin", 264)):
        b = nat.BlockEval.from_buffer_copy(a)
        setattr(b, field, bad)
        assert lib.yamb_block_eval_fwd(C.byref(b), st) == -1, field
        assert lib.yamb_last_error()
    b = nat.BlockEval.from_buffer_copy(a)
    b.Cout = 32                      # residual with Cin != Cout
    assert lib.yamb_block_eval_fwd(C.byref(b), st) == -1
    b = nat.BlockEval.from_buffer_copy(a)
    b.bn2.running_var = None
    assert lib.yamb_block_eval_fwd(C.byref(b), st) == -1
    b = nat.BlockEval.from_buffer_copy(a)
    b.w_expand = None                # no expansion needs Chid == Cin
    assert lib.yamb_block_eval_fwd(C.byref(b), st) == -1
    b = nat.BlockEval.from_buffer_copy(a)
    b.stride = 2                     # a skip connection needs stride 1
    assert lib.yamb_block_eval_fwd(C.byref(b), st) == -1


def test_mobilenet_v2_eval_uses_the_one_launch_blocks(built_lib):
    """Whole network, model.eval() under no_grad: all 17 blocks go through the one-launch
    kernel; logits against the reference graph in fp32 with the autocast yardstick."""
    import bench
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200 import engine
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda")
    model = bench.build_model()
    g = torch.Generator().manual_seed(11)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1, generator=g)
            m.running_var.uniform_(0.8, 1.25, generator=g)
    model = model.to(dev).eval()
    x = torch.randn(16, 3, 224, 224, generator=g).to(dev)
    c0 = engine.EVAL_FUSED_CALLS
    with torch.no_grad():
        y = model(x).float()
    torch.cuda.synchronize()
    assert engine.EVAL_FUSED_CALLS - c0 == 17
    ref = tm.as_reference(copy.deepcopy(model)).eval()
    with torch.no_grad():
        yt = ref(x)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ya = ref(x.contiguous(memory_format=torch.channels_last)).float()
    eo, ea = _rel(y, yt), _rel(ya, yt)
    assert eo <= SLACK * ea + FLOOR, (eo, ea)
    assert (y.argmax(1) == yt.argmax(1)).float().mean() > 0.8
