"""GPU parity of the eval path of InvertedResidualChannelsFused (engine.fused_class_eval_forward):
the one-launch block kernel with the Squeeze-and-Excitation gate (pool pass -> SE FCs -> block
kernel with the gate) and the non-local tail behind it (reference models/mobilenet_base.py:330-342
in model.eval() under torch.no_grad()).  Shapes from AutoNL-L and AtomNAS-C+ block 1.

Every case is checked against
  * the oracle with the kernel's rounding points (oracle.ir_block.forward(..., quant="fused")):
    rel-L2 < 3e-3;
  * fp32 truth from the stock-torch graph, with that graph under autocast-bf16 as the yardstick:
    err(ours) <= 1.5 * err(autocast) + 2.5e-3;
  * this repo's four-launch sequence: rel-L2 < 1e-2;
and must make exactly 1 C-ABI call (3 with SE, 4 more with a non-local block) and compute the
same bits twice.
"""
import copy
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

SLACK, FLOOR = 1.5, 2.5e-3


@pytest.fixture(autouse=True)
def every_covered_shape(monkeypatch):
    """Exercise the kernels on every shape they cover, including the ones the measured shape rule
    (engine.FUSED_CLASS_SHAPE_RULE) keeps on the four-launch sequence by default."""
    from yet_another_mobilenet_series_b200 import engine
    monkeypatch.setattr(engine, "FUSED_CLASS_SHAPE_RULE", False)


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _randomise(model, seed):
    """BatchNorm affine + running statistics (ZeroInitBN of the non-local block included: gamma = 0
    would switch the branch off), conv weights, SE biases."""
    g = torch.Generator().manual_seed(seed)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.weight.data.uniform_(0.5, 1.5, generator=g)
            m.bias.data.normal_(0, 0.3, generator=g)
            m.running_mean.normal_(0, 0.5, generator=g)
            m.running_var.uniform_(0.5, 2.0, generator=g)
        elif isinstance(m, torch.nn.Conv2d):
            fan = max(1, m.weight[0].numel())
            m.weight.data.normal_(0, (2.0 / fan) ** 0.5, generator=g)
            if m.bias is not None:
                m.bias.data.normal_(0, 0.5, generator=g)


def _make_block(cin, chid, cout, k, stride, expand, se, nl_c, nl_s, seed):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    torch.manual_seed(seed)
    blk = mb.InvertedResidualChannelsFused(
        cin, cout, stride, [chid], [k], expand, active_fn=mb.get_active_fn("nn.Swish"),
        batch_norm_kwargs={"momentum": 0.01, "eps": 1e-3}, se_ratio=0.25 if se else None,
        nl_c=nl_c, nl_s=nl_s)
    _randomise(blk, seed)
    return blk.eval()


# (cin, chid, cout, N, H, W, k, stride, expand, se, nl_c, nl_s)
CASES = [
    (80, 240, 80, 3, 14, 14, 3, 1, True, True, 0, 0),         # AutoNL-L block 10: SE alone
    (24, 72, 24, 3, 28, 28, 3, 1, True, False, 0.25, 2),      # block 4: non-local alone, nl_s 2
    (24, 144, 40, 2, 28, 28, 5, 2, True, False, 0.25, 1),     # block 5: non-local, nl_s 1, k5 s2
    (80, 240, 80, 3, 14, 14, 3, 1, True, True, 0.125, 2),     # block 12: SE + non-local
    (80, 480, 96, 2, 14, 14, 5, 1, True, True, 0.25, 1),      # block 13: SE + non-local, k5 s1
    (96, 288, 96, 3, 14, 14, 5, 1, True, True, 0, 0),         # block 14: Swish k5 s1
    (96, 576, 192, 2, 14, 14, 5, 2, True, True, 0.25, 1),     # block 17: Swish k5 s2
    (192, 1152, 320, 2, 7, 7, 5, 1, True, True, 0.25, 1),     # block 21: 1152 -> 320
    (40, 120, 40, 2, 13, 13, 7, 1, True, True, 0, 0),         # Swish k7, tiles overhang
    (40, 120, 80, 3, 13, 13, 7, 2, True, True, 0, 0),         # Swish k7 s2
    (32, 32, 16, 2, 112, 112, 3, 1, False, True, 0, 0),       # AtomNAS-C+ block 1: no expansion
    (96, 288, 96, 5, 7, 7, 5, 1, True, True, 0, 0),           # two images per tile, N odd
    (80, 240, 80, 3, 7, 7, 3, 1, True, True, 0.125, 2),       # two images per tile + non-local
    (24, 72, 24, 2, 19, 11, 5, 1, True, True, 0.25, 2),       # odd sizes, overhang, SE + non-local
    (16, 48, 24, 2, 23, 17, 5, 2, True, True, 0.25, 1),       # odd sizes, stride 2
]


def _case_id(c):
    return "x".join(str(v) for v in c)


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_fused_class_eval_block(built_lib, case):
    from oracle import ir_block as ob
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200 import engine
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cin, chid, cout, N, H, W, k, stride, expand, se, nl_c, nl_s = case
    dev = torch.device("cuda")
    blk = _make_block(cin, chid, cout, k, stride, expand, se, nl_c, nl_s, sum(case[:7]))
    g = torch.Generator().manual_seed(7)
    x = torch.randn(N, cin, H, W, generator=g).bfloat16().float()
    cfg, P = ob.extract(blk)
    yo, _ = ob.forward(x, cfg, P, training=False, quant="fused")
    blk_d = copy.deepcopy(blk).to(dev).eval()
    xd = x.to(dev)
    calls0, launches0 = engine.EVAL_FUSED_CALLS, engine.LAUNCHES
    with torch.no_grad():
        y = blk_d(xd)
    torch.cuda.synchronize()
    assert engine.EVAL_FUSED_CALLS == calls0 + 1, "the block did not take the eval path"
    assert engine.LAUNCHES - launches0 == 1 + (2 if se else 0) + (4 if nl_c else 0)
    assert y.shape == yo.shape and y.dtype == torch.bfloat16
    assert torch.isfinite(y.float()).all()
    with torch.no_grad():
        y2 = blk_d(xd)
    torch.cuda.synchronize()
    assert torch.equal(y, y2), "two runs differ"
    engine.EVAL_FUSED = False
    try:
        with torch.no_grad():
            y4 = blk_d(xd)
        torch.cuda.synchronize()
    finally:
        engine.EVAL_FUSED = True
    ref = tm.as_reference(copy.deepcopy(blk)).to(dev).eval()
    with torch.no_grad():
        yt = ref(xd)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ya = ref(xd.contiguous(memory_format=torch.channels_last))
    e_oracle, eo, ea, e4 = _rel(y, yo), _rel(y, yt), _rel(ya, yt), _rel(y, y4)
    print("%-40s vs oracle(fused points) %.3e | vs fp32 %.3e  autocast %.3e | vs four-launch "
          "%.3e" % (_case_id(case), e_oracle, eo, ea, e4))
    assert e_oracle < 3e-3, e_oracle
    assert eo <= SLACK * ea + FLOOR, (eo, ea)
    assert e4 < 1e-2, e4


def test_pool_pass_ignores_overhang_and_padding_image(built_lib):
    """yamb_block_eval_pool_fwd alone: the spatial mean of a2 against the oracle's, on a map the
    tiles overhang and an odd image count on the two-images-per-tile geometry."""
    from oracle import ir_block as ob
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200 import native as nat
    dev = torch.device("cuda")
    for (cin, chid, cout, N, H, W, k) in ((24, 72, 24, 3, 19, 11, 5), (96, 288, 96, 5, 7, 7, 5)):
        blk = _make_block(cin, chid, cout, k, 1, True, True, 0, 0, 11)
        x = torch.randn(N, cin, H, W).bfloat16().float()
        cfg, P = ob.extract(blk)
        _, S = ob.forward(x, cfg, P, training=False, quant="fused")
        bd = copy.deepcopy(blk).to(dev).eval()
        xd = engine.to_nhwc_bf16(x.to(dev))
        w1 = bd.expand_conv[0].weight.detach().flatten(1).to(torch.bfloat16).contiguous()
        w3 = bd.project_conv[0].weight.detach().flatten(1).to(torch.bfloat16).contiguous()
        stage = list(bd.depth_ops[0].children())[-1]
        a = engine._block_eval_args(bd, xd, None, w1, w3, stage[0],
                                    (bd.expand_conv[1], stage[1], bd.project_conv[1]), False)
        pooled = torch.full((N, chid), float("nan"), device=dev)
        a.pooled = pooled.data_ptr()
        nat.check(built_lib.yamb_block_eval_pool_fwd(ctypes.byref(a), nat.stream_handle()))
        torch.cuda.synchronize()
        assert torch.isfinite(pooled).all()
        assert _rel(pooled, S["se_s"]) < 1e-3, _rel(pooled, S["se_s"])


def _network(name, seed, x):
    """Model with non-zero ZeroInitBN gammas and SE biases, its BatchNorm running statistics
    calibrated on the batch x by the stock-torch graph (the reference's bn_calibration): with
    statistics of any other data the non-local products (cubic in their input) grow without bound
    through the 7x7 blocks of an untrained AutoNL-L."""
    from _cfg import build_from_cfg
    from oracle import torch_model as tm
    model, _ = build_from_cfg(name)
    g = torch.Generator().manual_seed(seed)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d) and float(m.weight.abs().sum()) == 0.0:
            m.weight.data.uniform_(0.05, 0.1, generator=g)         # ZeroInitBN of nl_op
        elif isinstance(m, torch.nn.Conv2d) and m.bias is not None:
            m.bias.data.normal_(0, 0.3, generator=g)                # SE biases
    ref = tm.as_reference(model).cuda().train()
    for m in ref.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.reset_running_stats()
            m.momentum = None
    with torch.no_grad():
        ref(x)
    model.load_state_dict({k: v.cpu() for k, v in ref.state_dict().items()})
    return model


@pytest.mark.parametrize("name,blocks", [("autonl_l", 21), ("atomnas_c+", 1)])
def test_network_eval(built_lib, name, blocks):
    """Whole network in eval() under no_grad: the number of blocks on this path, logits against
    the stock-torch graph in fp32 with the autocast yardstick."""
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200 import engine
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda")
    x = torch.randn(8, 3, 224, 224, generator=torch.Generator().manual_seed(3)).to(dev)
    model = _network(name, 5, x).to(dev).eval()
    c0 = engine.EVAL_FUSED_CALLS
    with torch.no_grad():
        y = model(x).float()
    torch.cuda.synchronize()
    assert engine.EVAL_FUSED_CALLS - c0 == blocks
    ref = tm.as_reference(copy.deepcopy(model)).eval()
    with torch.no_grad():
        yt = ref(x)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ya = ref(x.contiguous(memory_format=torch.channels_last)).float()
    eo, ea = _rel(y, yt), _rel(ya, yt)
    assert eo <= SLACK * ea + FLOOR, (eo, ea)


def test_autonl_eval_graph_replay_and_ema_copy(built_lib):
    """One AutoNL-L eval forward captured in a CUDA graph and replayed computes the eager bits;
    a deepcopy of the model taken after an eval forward (the EMA model) computes them too."""
    from yet_another_mobilenet_series_b200 import engine
    dev = torch.device("cuda")
    x = torch.randn(4, 3, 224, 224, generator=torch.Generator().manual_seed(4)).to(dev)
    model = _network("autonl_l", 9, x).to(dev).eval()
    with torch.no_grad():
        y_eager = model(x).clone()
        ema = copy.deepcopy(model)
        c0 = engine.EVAL_FUSED_CALLS
        y_ema = ema(x)
        assert engine.EVAL_FUSED_CALLS - c0 == 21
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            model(x)                                   # warm-up on the capture stream
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            y_static = model(x)
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(y_ema, y_eager)
    assert torch.equal(y_static, y_eager)
