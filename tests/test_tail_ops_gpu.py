"""GPU parity of the layers around the block stack on the sm_90a path (tail_ops.py): stem 3x3/s2
convolution, head 1x1 ConvBNReLU and classifier through the wgmma GEMM, label-smoothed softmax
cross entropy with top-k.  Truth = the reference's stock-torch modules / formulas in fp32 on the
same bf16-rounded inputs (reference models/mobilenet_supernet.py:124-130, :152-167,
models/mobilenet_base.py:181-203, utils/optim.py:150-158, common.py:73-79)."""
import copy

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _bn_randomise(m, g):
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.weight.data.uniform_(0.5, 1.5, generator=g)
            mod.bias.data.normal_(0, 0.3, generator=g)


# (640, 2560): the head of a width-2.0 network (last_channel = 1280 * width_mult)
@pytest.mark.parametrize("cin,cout,hw,act", [(320, 1280, 7, "nn.ReLU"), (64, 136, 5, "nn.Swish"),
                                             (640, 2560, 7, "nn.ReLU")])
def test_head_pointwise_conv_bn_act(built_lib, cin, cout, hw, act):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(1)
    bnk = {"momentum": 0.01, "eps": 1e-3}
    mod = mb.ConvBNReLU(cin, cout, kernel_size=1, batch_norm_kwargs=bnk, active_fn=mb.get_active_fn(act))
    mod.apply(mb.init_weights_mnas)
    _bn_randomise(mod, g)
    ref = torch.nn.Sequential(*copy.deepcopy(list(mod))).cuda().train()   # plain nn.Sequential
    mod = mod.cuda().train()
    x = torch.randn(32, cin, hw, hw, generator=g).bfloat16().float().cuda()
    dy = torch.randn(32, cout, hw, hw, generator=g).bfloat16().float().cuda()
    xr = x.clone().requires_grad_(True)
    yr = ref(xr)
    yr.backward(dy)
    # yardstick: the same stock modules under autocast-bf16, channels_last (SURVEY.md 8c gate ii)
    yard = copy.deepcopy(ref)
    for q in yard.parameters():
        q.grad = None
    xa = x.clone().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        ya = yard.to(memory_format=torch.channels_last)(xa)
    ya.backward(dy.to(ya.dtype))
    xo = x.clone().requires_grad_(True)
    yo = mod(xo)
    assert yo.dtype == torch.bfloat16
    yo.backward(dy.to(yo.dtype))
    torch.cuda.synchronize()

    def gate(o, a, t, what):
        eo, ea = _rel(o, t), _rel(a, t)
        assert eo <= 1.5 * ea + 2.5e-3, (what, eo, ea)

    gate(yo, ya, yr, "y")
    gate(xo.grad, xa.grad, xr.grad, "dx")
    gate(mod[0].weight.grad, yard[0].weight.grad, ref[0].weight.grad, "dW")
    gate(mod[1].weight.grad, yard[1].weight.grad, ref[1].weight.grad, "dgamma")
    gate(mod[1].bias.grad, yard[1].bias.grad, ref[1].bias.grad, "dbeta")
    assert _rel(mod[1].running_mean, ref[1].running_mean) < 5e-3
    assert _rel(mod[1].running_var, ref[1].running_var) < 5e-3
    assert int(mod[1].num_batches_tracked) == 1
    # eval mode: running statistics, no update
    mod.eval(), ref.eval()
    with torch.no_grad():
        assert _rel(mod(x), ref(x)) < 6e-3
    assert int(mod[1].num_batches_tracked) == 1


@pytest.mark.parametrize("layer", ["head", "stem"])
def test_backward_reads_its_own_forward_statistics(built_lib, layer):
    """Forward A, forward B on another batch, then A's backward: dx and the parameter gradients
    equal, bit for bit, those of a copy that ran A's forward and backward alone (the BatchNorm
    backward reads the statistics its own forward took, not those of the latest forward).  As in
    training, the parameters live in the fused optimizer's flat arena: the head's bf16 weight
    operand is the optimizer's mirror, which forward B leaves alone (forward B rewrites a
    module-owned copy, and autograd then refuses A's backward)."""
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    from yet_another_mobilenet_series_b200.fused_rmsprop import RMSprop
    g = torch.Generator().manual_seed(6)
    bnk = {"momentum": 0.01, "eps": 1e-3}
    relu = mb.get_active_fn("nn.ReLU")
    # module construction draws from the global generator: leave it as the later tests find it
    with torch.random.fork_rng(devices=[]):
        if layer == "head":
            mod = mb.ConvBNReLU(320, 1280, kernel_size=1, batch_norm_kwargs=bnk, active_fn=relu)
            shape = (16, 320, 7, 7)
        else:
            mod = mb.ConvBNReLU(3, 32, stride=2, batch_norm_kwargs=bnk, active_fn=relu)
            shape = (4, 3, 64, 64)
        mod.apply(mb.init_weights_mnas)
    _bn_randomise(mod, g)
    alone = copy.deepcopy(mod).cuda().train()
    mod = mod.cuda().train()
    opts = [RMSprop(m.parameters(), lr=0.016, alpha=0.9, momentum=0.9, eps=1e-3,
                    eps_inside_sqrt=True) for m in (alone, mod)]
    for o in opts:
        o.arenas()
    xa = torch.randn(shape, generator=g).cuda()
    xb = (torch.randn(shape, generator=g) * 3 + 1).cuda()

    def grads(m, others):
        x = xa.clone().requires_grad_(layer == "head")     # the stem has no input gradient
        y = m(x)
        for o in others:
            m(o)
        y.backward(torch.randn(y.shape, generator=torch.Generator().manual_seed(7)).cuda()
                   .to(y.dtype))
        torch.cuda.synchronize()
        return ([x.grad] if layer == "head" else []) + [p.grad for p in m.parameters()]

    want = grads(alone, [])
    got = grads(mod, [xb])
    assert len(got) == len(want) == (4 if layer == "head" else 3)
    for a, b in zip(got, want):
        assert torch.equal(a, b)


def test_classifier_linear(built_lib):
    from yet_another_mobilenet_series_b200 import tail_ops
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator().manual_seed(2)
    lin = torch.nn.Linear(1280, 1000)
    ref = copy.deepcopy(lin).cuda()
    lin = lin.cuda()
    x = (torch.randn(256, 1280, generator=g) * 0.5).bfloat16().float().cuda()
    dy = (torch.randn(256, 1000, generator=g) * 1e-2).bfloat16().float().cuda()
    xr = x.clone().requires_grad_(True)
    ref(xr).backward(dy)
    xo = x.clone().requires_grad_(True)
    assert tail_ops.linear_supported(lin, xo)
    y = tail_ops.linear_apply(lin, xo)
    y.backward(dy.to(y.dtype))
    torch.cuda.synchronize()
    assert _rel(y, ref(x)) < 5e-3
    assert _rel(xo.grad, xr.grad) < 1e-2
    assert _rel(lin.weight.grad, ref.weight.grad) < 1e-2
    assert _rel(lin.bias.grad, ref.bias.grad) < 1e-2


@pytest.mark.parametrize("N,C", [(256, 1000), (7, 10)])
def test_softmax_ce_topk(built_lib, N, C):
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200 import tail_ops
    g = torch.Generator().manual_seed(3)
    logits = (torch.randn(N, C, generator=g) * 3).bfloat16().float()
    target = torch.randint(0, C, (N,), generator=g)
    lo = logits.cuda().requires_grad_(True)
    loss, c1, c5 = tail_ops.softmax_ce(lo, target.cuda(), 0.1)
    w = torch.randn(N, generator=g).cuda()
    (loss * w).sum().backward()
    torch.cuda.synchronize()
    lr = logits.double().requires_grad_(True)
    want = tm.label_smooth_ce(lr, target, 0.1)       # utils/optim.py:150-158 restated
    (want * w.cpu().double()).sum().backward()
    assert _rel(loss, want) < 2e-6
    _, pred = logits.topk(min(5, C))                 # common.py:73-79
    corr = pred.t().eq(target.view(1, -1).expand_as(pred.t()))
    assert torch.equal(c1.cpu(), corr[:1].float().sum(0))
    assert torch.equal(c5.cpu(), corr[:5].float().sum(0))
    assert _rel(lo.grad, lr.grad) < 4e-3             # bf16 storage of softmax - target
    # ties (torch.topk leaves their order unspecified): here the lower class index ranks first
    tie = torch.full((2, C), 0.25)
    tt = torch.tensor([min(4, C - 1), min(5, C - 1)])
    _, t1, t5 = tail_ops.softmax_ce(tie.cuda(), tt.cuda(), 0.1)
    assert t1.cpu().tolist() == [0.0, 0.0]
    assert t5.cpu().tolist() == ([1.0, 0.0] if C > 5 else [1.0, 1.0])


def test_stem_conv(built_lib):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    torch.backends.cudnn.allow_tf32 = False
    g = torch.Generator().manual_seed(4)
    bnk = {"momentum": 0.01, "eps": 1e-3}
    for cout, hw, n in ((32, 224, 4), (16, 37, 3)):          # odd size: partial tiles, borders
        mod = mb.ConvBNReLU(3, cout, stride=2, batch_norm_kwargs=bnk,
                            active_fn=mb.get_active_fn("nn.ReLU"))
        mod.apply(mb.init_weights_mnas)
        _bn_randomise(mod, g)
        ref = torch.nn.Sequential(*copy.deepcopy(list(mod))).cuda().train()
        mod = mod.cuda().train()
        x = torch.randn(n, 3, hw, hw, generator=g).bfloat16().float().cuda()
        yr = ref(x)
        dy = torch.randn(yr.shape, generator=g).bfloat16().float().cuda()
        yr.backward(dy)
        yo = mod(x)
        yo.backward(dy.to(yo.dtype))
        torch.cuda.synchronize()
        assert yo.shape == yr.shape
        assert _rel(yo, yr) < 6e-3, (cout, hw)
        assert _rel(mod[0].weight.grad, ref[0].weight.grad) < 2e-2, (cout, hw)
        assert _rel(mod[1].weight.grad, ref[1].weight.grad) < 2e-2
        assert _rel(mod[1].running_var, ref[1].running_var) < 5e-3


_STEM_CHILD = r"""
import ctypes as C, sys
import torch
sys.path.insert(0, sys.argv[1])
from yet_another_mobilenet_series_b200 import native as nat

def stem(cout, fwd):
    # 64 x 224 x 224: 1792 tiles, more than one resident wave, so the wgrad grid (and with it the
    # partial slabs and the order of their sum) is the occupancy at this Cout's shared memory
    g = torch.Generator().manual_seed(cout)
    N, H, W, Ho, Wo = 64, 224, 224, 112, 112
    x = torch.randn(N, H, W, 3, generator=g).bfloat16().cuda()
    w = torch.randn(cout, 3, 3, 3, generator=g).cuda()
    dh = torch.randn(N, Ho, Wo, cout, generator=g).bfloat16().cuda()
    y = torch.empty(N, Ho, Wo, cout, dtype=torch.bfloat16, device="cuda")
    dw = torch.zeros(cout, 3, 3, 3, device="cuda")
    a = nat.StemConv()
    a.N, a.H, a.W, a.Cout = N, H, W, cout
    a.x, a.w, a.y, a.dh, a.dw = x.data_ptr(), w.data_ptr(), y.data_ptr(), dh.data_ptr(), dw.data_ptr()
    if fwd:
        nat.check(nat.lib().yamb_stem_conv_fwd(C.byref(a), nat.stream_handle()))
    nat.check(nat.lib().yamb_stem_conv_wgrad(C.byref(a), nat.stream_handle()))
    torch.cuda.synchronize()
    return dw

if sys.argv[3] == "after16":
    stem(16, True)
print(stem(int(sys.argv[2]), False).cpu().numpy().tobytes().hex())
"""


# on an H100 the wgrad kernel has 3 CTAs per SM at Cout = 16 and 32 (registers), 2 at Cout = 64
# (shared memory)
@pytest.mark.parametrize("cout", [32, 64])
def test_stem_wgrad_bits_do_not_depend_on_earlier_widths(built_lib, cout):
    """The stem weight gradient at `cout` in a fresh process, and in one that first ran the stem
    at Cout = 16: each width's grid comes from its own occupancy, so the bits are the same."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _STEM_CHILD, root,
                                                                           str(cout)]
    out = {}
    for order in ("fresh", "after16"):
        r = subprocess.run(cmd + [order], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-4000:]
        out[order] = r.stdout.strip().splitlines()[-1]
    assert len(out["fresh"]) == 2 * 4 * cout * 27
    assert out["fresh"] == out["after16"]


def test_data_prefetcher_surface_and_values(built_lib):
    """DataPrefetcher (reference utils/dataflow.py:13-58): iterator surface, device placement,
    bf16 channels_last conversion, buffer recycling without tearing."""
    from yet_another_mobilenet_series_b200.dataflow import DataPrefetcher
    g = torch.Generator().manual_seed(5)
    batches = [(torch.randn(4, 3, 32, 32, generator=g).pin_memory(),
                torch.randint(0, 10, (4,), generator=g).pin_memory()) for _ in range(5)]
    pf = DataPrefetcher(batches)
    assert len(pf) == 5
    seen = 0
    acc = []
    for (x, t), (hx, ht) in zip(pf, batches):
        assert x.is_cuda and x.dtype == torch.bfloat16
        assert x.is_contiguous(memory_format=torch.channels_last)
        acc.append((x.float().sum(), hx.bfloat16().float().sum()))   # consumed before the next batch
        assert torch.equal(t.cpu(), ht)
        seen += 1
    assert seen == 5
    torch.cuda.synchronize()
    for a, b in acc:
        assert abs(float(a) - float(b)) < 1e-2 * (abs(float(b)) + 1.0)
