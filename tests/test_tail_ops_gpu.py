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


@pytest.mark.parametrize("cin,cout,hw,act", [(320, 1280, 7, "nn.ReLU"), (64, 136, 5, "nn.Swish")])
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
