"""GPU parity of the cluster split of the one-launch eval block (yamb_block_eval_cluster_fwd /
yamb_block_eval_cluster_pool_fwd): the hidden slices of every output tile spread over the CTAs of
a thread-block cluster, the fp32 project partials added in rank order over distributed shared
memory.

Every case of tests/test_block_eval_gpu.py plus every MobileNetV2 and Proxyless-mobile block at
N = 1, 2, 3 runs with the cluster size forced to 1 (the unsplit kernel), 2, 4 and 8 where the
hidden dimension has that many 64-channel slices, each checked against
  * the oracle with the kernel's rounding points (oracle.ir_block.forward(..., quant="fused")):
    rel-L2 < 3e-3;
  * fp32 truth from the stock-torch graph with that graph under autocast-bf16 as the yardstick:
    err(ours) <= 1.5 * err(autocast) + 2.5e-3;
  * the same bits on a second run, and from a CUDA graph replay.
The SE gate and pool passes run on AutoNL-L's 3x3 SE blocks; whole networks run through EvalStep
at N = 1 and 4.
"""
import copy

import pytest
import torch

from test_block_eval_gpu import CASES as BLOCK_CASES
from test_block_eval_gpu import _make_block
from test_fused_class_eval_gpu import _make_block as _make_fused_block

pytestmark = pytest.mark.gpu

SLACK, FLOOR = 1.5, 2.5e-3
SIZES = (1, 2, 4, 8)

# (cin, chid, cout, H, stride, k, expand) of every block, 224 input
MBV2 = [(32, 32, 16, 112, 1, 3, False), (16, 96, 24, 112, 2, 3, True), (24, 144, 24, 56, 1, 3, True),
        (24, 144, 32, 56, 2, 3, True), (32, 192, 32, 28, 1, 3, True), (32, 192, 64, 28, 2, 3, True),
        (64, 384, 64, 14, 1, 3, True), (64, 384, 96, 14, 1, 3, True), (96, 576, 96, 14, 1, 3, True),
        (96, 576, 160, 14, 2, 3, True), (160, 960, 160, 7, 1, 3, True),
        (160, 960, 320, 7, 1, 3, True)]
PROXYLESS = [(32, 32, 16, 112, 1, 3, False), (16, 48, 32, 112, 2, 5, True),
             (32, 96, 32, 56, 1, 3, True), (32, 96, 40, 56, 2, 7, True),
             (40, 120, 40, 28, 1, 3, True), (40, 120, 40, 28, 1, 5, True),
             (40, 240, 80, 28, 2, 7, True), (80, 240, 80, 14, 1, 5, True),
             (80, 480, 96, 14, 1, 5, True), (96, 288, 96, 14, 1, 5, True),
             (96, 576, 192, 14, 2, 7, True), (192, 1152, 192, 7, 1, 7, True),
             (192, 576, 192, 7, 1, 7, True), (192, 1152, 320, 7, 1, 7, True)]
NET_CASES = [(cin, chid, cout, n, h, h, "relu6", s, ex, k)
             for cin, chid, cout, h, s, k, ex in sorted(set(MBV2 + PROXYLESS)) for n in (1, 2, 3)]


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _case_id(c):
    return "x".join(str(v) for v in c)


def _sizes(chid):
    return [s for s in SIZES if s <= (chid + 63) // 64]


def _run(engine, blk_d, xd, cluster):
    engine.EVAL_CLUSTER = cluster
    try:
        with torch.no_grad():
            y = blk_d(xd)
        torch.cuda.synchronize()
    finally:
        engine.EVAL_CLUSTER = None
    return y


@pytest.mark.parametrize("case", BLOCK_CASES + NET_CASES, ids=_case_id)
def test_cluster_eval_block(built_lib, case):
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
    x = torch.randn(N, cin, H, W, generator=torch.Generator().manual_seed(7)).bfloat16().float()
    cfg, P = ob.extract(blk)
    yo, _ = ob.forward(x, cfg, P, training=False, quant="fused")
    blk_d = copy.deepcopy(blk).to(dev).eval()
    xd = x.to(dev)
    ref = tm.as_reference(copy.deepcopy(blk)).to(dev).eval()
    with torch.no_grad():
        yt = ref(xd)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ya = ref(xd.contiguous(memory_format=torch.channels_last))
    ea = _rel(ya, yt)
    for s in _sizes(chid):
        c0, l0 = engine.EVAL_CLUSTER_CALLS, engine.LAUNCHES
        y = _run(engine, blk_d, xd, s)
        assert engine.LAUNCHES == l0 + 1
        split = engine.EVAL_CLUSTER_CALLS - c0
        if s > 1 and not split:   # refused: only a tile plan that does not fit shared memory
            assert b"shared memory" in built_lib.yamb_last_error(), built_lib.yamb_last_error()
        assert torch.isfinite(y.float()).all()
        assert torch.equal(y, _run(engine, blk_d, xd, s)), "two runs differ (S = %d)" % s
        e_oracle, eo = _rel(y, yo), _rel(y, yt)
        print("%-34s S=%d%s vs oracle %.3e | vs fp32 %.3e autocast %.3e"
              % (_case_id(case), s, "" if split or s == 1 else " (unsplit: no fit)",
                 e_oracle, eo, ea))
        assert e_oracle < 3e-3, (s, e_oracle)
        assert eo <= SLACK * ea + FLOOR, (s, eo, ea)


# AutoNL-L 3x3 SE blocks (Swish): the pool pass and the gated block kernel, split and unsplit;
# (cin, chid, cout, N, H, stride): 4 slices (block 10 at 14x14 and 28x28), a residual, stride 2
SE_CASES = [(80, 240, 80, 1, 14, 1), (80, 240, 80, 3, 14, 1), (40, 120, 40, 2, 28, 1),
            (40, 240, 80, 1, 28, 2), (96, 576, 96, 1, 14, 1)]


@pytest.mark.parametrize("case", SE_CASES, ids=_case_id)
def test_cluster_se_gate_and_pool(built_lib, case):
    from oracle import ir_block as ob
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200 import engine
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cin, chid, cout, N, H, stride = case
    dev = torch.device("cuda")
    blk = _make_fused_block(cin, chid, cout, 3, stride, True, True, 0, 0, sum(case))
    x = torch.randn(N, cin, H, H, generator=torch.Generator().manual_seed(9)).bfloat16().float()
    cfg, P = ob.extract(blk)
    yo, _ = ob.forward(x, cfg, P, training=False, quant="fused")
    blk_d = copy.deepcopy(blk).to(dev).eval()
    xd = x.to(dev)
    ref = tm.as_reference(copy.deepcopy(blk)).to(dev).eval()
    with torch.no_grad():
        yt = ref(xd)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ya = ref(xd.contiguous(memory_format=torch.channels_last))
    ea = _rel(ya, yt)
    for s in _sizes(chid):
        c0 = engine.EVAL_CLUSTER_CALLS
        y = _run(engine, blk_d, xd, s)
        assert engine.EVAL_CLUSTER_CALLS - c0 == (2 if s > 1 else 0)   # pool pass + gated kernel
        assert torch.equal(y, _run(engine, blk_d, xd, s))
        assert _rel(y, yo) < 3e-3, (s, _rel(y, yo))
        assert _rel(y, yt) <= SLACK * ea + FLOOR, (s, _rel(y, yt), ea)


def test_cluster_pool_pass_equals_unsplit(built_lib):
    """The pool pass writes the same means split or not: each rank pools its own slices."""
    import ctypes
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200 import native as nat
    dev = torch.device("cuda")
    blk = _make_fused_block(80, 240, 80, 3, 1, True, True, 0, 0, 3).to(dev)
    xd = engine.to_nhwc_bf16(torch.randn(2, 80, 14, 14, device=dev))
    w1 = blk.expand_conv[0].weight.detach().flatten(1).to(torch.bfloat16).contiguous()
    w3 = blk.project_conv[0].weight.detach().flatten(1).to(torch.bfloat16).contiguous()
    stage = list(blk.depth_ops[0].children())[-1]
    a = engine._block_eval_args(blk, xd, None, w1, w3, stage[0],
                                (blk.expand_conv[1], stage[1], blk.project_conv[1]), False)
    outs = []
    for s in (1, 2, 4):
        pooled = torch.full((2, 240), float("nan"), device=dev)
        a.pooled = pooled.data_ptr()
        st = nat.stream_handle()
        rc = built_lib.yamb_block_eval_pool_fwd(ctypes.byref(a), st) if s == 1 else \
            built_lib.yamb_block_eval_cluster_pool_fwd(ctypes.byref(a), s, st)
        nat.check(rc)
        torch.cuda.synchronize()
        outs.append(pooled)
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


def test_cluster_graph_replay_equals_eager(built_lib):
    from yet_another_mobilenet_series_b200 import engine
    dev = torch.device("cuda")
    blk = _make_block(160, 960, 160, "relu", 5).to(dev)
    x = torch.randn(1, 160, 7, 7, device=dev).to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last)
    y0 = _run(engine, blk, x, None)
    assert engine.eval_cluster_size(3, 1, 1, 7, 7, 960, 160,
                                    torch.cuda.get_device_properties(dev).multi_processor_count) == 8
    with torch.no_grad():
        blk(x)
        g = torch.cuda.CUDAGraph()
        c0 = engine.EVAL_CLUSTER_CALLS
        with torch.cuda.graph(g):
            yg = blk(x)
        assert engine.EVAL_CLUSTER_CALLS == c0 + 1
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(yg, y0)


def test_cluster_abi_rejects(built_lib):
    import ctypes as C
    from yet_another_mobilenet_series_b200 import native as nat
    lib = built_lib
    dev = torch.device("cuda")
    buf = torch.zeros(1 << 16, device=dev, dtype=torch.float32)
    a = nat.BlockEval()
    a.N, a.H, a.W, a.Cin, a.Chid, a.Cout = 1, 8, 8, 16, 256, 16
    a.kernel, a.stride, a.act, a.residual = 3, 1, 1, 1
    for f in ("x", "y", "w_expand", "w_dw", "w_project"):
        setattr(a, f, buf.data_ptr())
    for bn in (a.bn1, a.bn2, a.bn3):
        bn.running_mean = bn.running_var = buf.data_ptr()
        bn.eps = 1e-3
    st = torch.cuda.current_stream().cuda_stream
    for cs in (2, 4, 8):
        assert lib.yamb_block_eval_cluster_fwd(C.byref(a), cs, st) == 0
    torch.cuda.synchronize()
    for cs in (0, 1, 3, 16):
        assert lib.yamb_block_eval_cluster_fwd(C.byref(a), cs, st) == -1
    b = nat.BlockEval.from_buffer_copy(a)
    b.Cout = 328
    assert lib.yamb_block_eval_cluster_fwd(C.byref(b), 2, st) == -1


NETWORKS = ["mobilenet_v2", "proxyless_mobile", "autonl_l"]


@pytest.mark.parametrize("name", NETWORKS)
@pytest.mark.parametrize("batch", [1, 4])
def test_cluster_eval_step_network(built_lib, name, batch):
    """EvalStep at a small batch (one captured graph with the split launches inside): logits
    against the stock-torch graph in fp32 with the autocast yardstick, and against the unsplit
    path."""
    from oracle import torch_model as tm
    from test_fused_class_eval_gpu import _network
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import EvalStep
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda")
    x = torch.randn(batch, 3, 224, 224, generator=torch.Generator().manual_seed(3))
    t = torch.zeros(batch, dtype=torch.long)
    model = _network(name, 4, torch.randn(16, 3, 224, 224).to(dev)).to(dev).eval()
    logits = {}
    for cluster in (None, 1):
        es = EvalStep(copy.deepcopy(model), batch, use_graph=True)
        engine.EVAL_CLUSTER = cluster
        try:
            c0 = engine.EVAL_CLUSTER_CALLS
            for _ in range(3):            # eager warm-up, capture + replay, replay
                es.evaluate([(x.bfloat16(), t)])
            assert es.phases["eval"].graph is not None
            split = engine.EVAL_CLUSTER_CALLS - c0
        finally:
            engine.EVAL_CLUSTER = None
        torch.cuda.synchronize()
        assert (split > 0) == (cluster is None), split
        logits[cluster] = es.logits.float().clone()
    ref = tm.as_reference(copy.deepcopy(model)).eval()
    with torch.no_grad():
        xr = x.bfloat16().float().to(dev)
        yt = ref(xr).float()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ya = ref(xr.contiguous(memory_format=torch.channels_last)).float()
    eo, ea, eu = _rel(logits[None], yt), _rel(ya, yt), _rel(logits[None], logits[1])
    print("%s N=%d: split vs fp32 %.3e, autocast %.3e, vs unsplit %.3e" % (name, batch, eo, ea, eu))
    assert eo <= SLACK * ea + FLOOR, (eo, ea)
    assert eu <= 2 * (SLACK * ea + FLOOR), (eu, ea)     # both within the yardstick of fp32
