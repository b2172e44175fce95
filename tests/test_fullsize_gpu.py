"""GPU parity AT THE BENCHMARK SHAPES (VERDICT r1, "parity is proven only on toy shapes").

Every one of the 17 inverted-residual blocks of MobileNetV2-1.0 (SURVEY.md §8d: 224x224-derived
spatial sizes 112^2 .. 7^2; reference models/mobilenet_base.py:446-451 built by
models/mobilenet_supernet.py:132-149 from apps/mobilenet/mobilenet_v2_mnas.yml) runs through the
sm_90a kernel sequence at N = 32, and blocks 1-3 also at the bench batch N = 256 (M = 3.2 M
pixels, split-K wgrad over K = 3.2 M), against

  truth      the reference's stock-torch graph of the same block in fp32 on the same GPU
             (oracle.torch_model.as_reference, TF32 off), and
  yardstick  the SAME graph under torch.autocast(bfloat16), channels_last — "the reference's own
             bf16 path" — measured in the same run (SURVEY.md §8c gate ii).

Gate: for y, dx, EVERY parameter gradient and every BatchNorm running statistic, the rel-L2 error
of this path against the truth is no larger than SLACK x the yardstick's error (+ a floor at the
bf16 output-rounding level).  The measured table is written to gpurun_out/fullsize_parity.txt.
"""
import copy
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SLACK = 1.5        # ours <= SLACK * autocast-yardstick + FLOOR
FLOOR = 2.5e-3     # bf16 output rounding alone is 1.65e-3 rel-L2 (SURVEY §8c)


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _mbv2_blocks():
    import bench
    model = bench.build_model()
    blocks = [m for m in model.features if hasattr(m, "pw_bn")]
    assert len(blocks) == 17
    return blocks


def _input_hw(idx):
    # spatial size of the INPUT of block idx (0-based) at 224x224
    sizes = [112, 112, 56, 56, 28, 28, 28, 14, 14, 14, 14, 14, 14, 14, 7, 7, 7]
    return sizes[idx]


CASES = [(i, 32) for i in range(17)] + [(0, 256), (1, 256), (2, 256)]


@pytest.mark.parametrize("idx,N", CASES)
def test_mbv2_block_fullsize_vs_fp32_and_autocast(built_lib, idx, N):
    from oracle import torch_model as tm
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda")
    blk = copy.deepcopy(_mbv2_blocks()[idx])
    g = torch.Generator().manual_seed(100 + idx)
    for m in blk.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.weight.data.uniform_(0.5, 1.5, generator=g)
            m.bias.data.normal_(0, 0.3, generator=g)
    hw = _input_hw(idx)
    x = torch.randn(N, blk.input_dim, hw, hw, generator=g).bfloat16().float()
    ho = (hw - 1) // blk.stride + 1
    dy = torch.randn(N, blk.output_dim, ho, ho, generator=g).bfloat16().float()

    def run(mod, xin, dyin, autocast):
        mod = mod.to(dev).train()
        xi = xin.to(dev).requires_grad_(True)
        if autocast:
            with torch.autocast("cuda", dtype=torch.bfloat16):
                y = mod(xi.contiguous(memory_format=torch.channels_last))
        else:
            y = mod(xi)
        y.backward(dyin.to(dev).to(y.dtype))
        torch.cuda.synchronize()
        grads = {k: p.grad.detach().float().cpu() for k, p in mod.named_parameters()}
        stats = {k: v.detach().float().cpu() for k, v in mod.named_buffers() if "running_" in k}
        return y.detach().float().cpu(), xi.grad.detach().float().cpu(), grads, stats

    truth = run(tm.as_reference(blk), x, dy, False)
    yard = run(tm.as_reference(blk), x, dy, True)
    ours = run(blk, x, dy, False)
    assert ours[0].shape == truth[0].shape
    rows, bad = [], []

    def gate(name, o, a, t):
        eo, ea = _rel(o, t), _rel(a, t)
        rows.append("%-34s ours %.3e  autocast %.3e  ratio %.2f" % (name, eo, ea, eo / max(ea, 1e-12)))
        if not eo <= SLACK * ea + FLOOR:
            bad.append(rows[-1])

    gate("y", ours[0], yard[0], truth[0])
    gate("dx", ours[1], yard[1], truth[1])
    for k in truth[2]:
        gate("grad " + k, ours[2][k], yard[2][k], truth[2][k])
    for k in truth[3]:
        gate("stat " + k, ours[3][k], yard[3][k], truth[3][k])
    out = os.path.join(ROOT, "gpurun_out")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "fullsize_parity.txt"), "a") as f:
        f.write("== MobileNetV2 block %d  N=%d  %dx%d  %s\n" % (idx + 1, N, hw, hw, blk))
        f.write("\n".join(rows) + "\n")
    assert not bad, "\n".join(bad)


# ---- the other BASELINE.json configurations: a sample of their REAL blocks at 224x224-derived
# sizes (multi-branch k in {3,5,7}, odd AtomNAS widths through the padded shadow, SE + Swish,
# non-local blocks), same truth / yardstick / gate as above ----------------------------------------
def _cfg_blocks(name):
    from _cfg import build_from_cfg
    model, _ = build_from_cfg(name)
    blocks, hw = [], 112
    for m in model.features:
        if hasattr(m, "channels") and hasattr(m, "use_res_connect"):
            blocks.append((m, hw))
            hw = (hw - 1) // m.stride + 1
    return blocks


CFG_CASES = [("proxyless_mobile", i) for i in (1, 4, 9, 13, 19)] + \
            [("atomnas_c+", i) for i in (1, 5, 10, 16, 21)] + \
            [("autonl_l", i) for i in (1, 3, 8, 12, 20)]


@pytest.mark.parametrize("cfg,idx", CFG_CASES)
def test_config_block_fullsize_vs_fp32_and_autocast(built_lib, cfg, idx):
    from oracle import torch_model as tm
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda")
    N = 32
    blocks = _cfg_blocks(cfg)
    blk, hw = blocks[min(idx, len(blocks) - 1)]
    blk = copy.deepcopy(blk)
    g = torch.Generator().manual_seed(500 + idx)
    for m in blk.modules():
        if isinstance(m, torch.nn.BatchNorm2d):      # incl. the non-local block's ZeroInitBN
            m.weight.data.uniform_(0.5, 1.5, generator=g)
            m.bias.data.normal_(0, 0.3, generator=g)
    x = torch.randn(N, blk.input_dim, hw, hw, generator=g).bfloat16().float()
    ho = (hw - 1) // blk.stride + 1
    dy = torch.randn(N, blk.output_dim, ho, ho, generator=g).bfloat16().float()
    if getattr(blk, "nl_c", 0):
        x = x * 0.25        # the non-local product grows with the cube of the activations

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
        return (y.detach().float().cpu(), xi.grad.detach().float().cpu(),
                {k: p.grad.detach().float().cpu() for k, p in mod.named_parameters()},
                {k: v.detach().float().cpu() for k, v in mod.named_buffers() if "running_" in k})

    truth = run(tm.as_reference(blk), False)
    yard = run(tm.as_reference(blk), True)
    ours = run(blk, False)
    rows, bad = [], []

    def gate(name, o, a, t):
        eo, ea = _rel(o, t), _rel(a, t)
        rows.append("%-40s ours %.3e  autocast %.3e  ratio %.2f" % (name, eo, ea, eo / max(ea, 1e-12)))
        if not eo <= SLACK * ea + FLOOR:
            bad.append(rows[-1])

    gate("y", ours[0], yard[0], truth[0])
    gate("dx", ours[1], yard[1], truth[1])
    for k in truth[2]:
        gate("grad " + k, ours[2][k], yard[2][k], truth[2][k])
    for k in truth[3]:
        gate("stat " + k, ours[3][k], yard[3][k], truth[3][k])
    out = os.path.join(ROOT, "gpurun_out")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "fullsize_parity.txt"), "a") as f:
        f.write("== %s block %d  N=%d  %dx%d  %s\n" % (cfg, idx, N, hw, hw, blk))
        f.write("\n".join(rows) + "\n")
    assert not bad, "\n".join(bad)
