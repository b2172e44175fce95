"""Stand-alone BatchNorm+activation kernels behind a torch convolution (stem / head ConvBNReLU,
reference models/mobilenet_base.py:181-203) against torch's own BatchNorm2d + activation."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-20))


@pytest.mark.parametrize("C,H,act,train", [(32, 24, "ReLU6", True), (1280, 3, "ReLU", True),
                                           (64, 9, "Swish", True), (32, 16, "ReLU6", False),
                                           (2048, 3, "ReLU", True)])
def test_bn_act_matches_torch(built_lib, C, H, act, train):
    from yet_another_mobilenet_series_b200 import engine, mobilenet_base as mb
    torch.manual_seed(0)
    dev = "cuda"
    N = 4
    bn = torch.nn.BatchNorm2d(C, momentum=0.01, eps=1e-3).to(dev)
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.normal_(0, 0.3)
        bn.running_mean.normal_(0, 0.2)
        bn.running_var.uniform_(0.5, 1.5)
    ref = torch.nn.BatchNorm2d(C, momentum=0.01, eps=1e-3).to(dev)
    ref.load_state_dict(bn.state_dict())
    bn.train(train)
    ref.train(train)
    actm = {"ReLU6": torch.nn.ReLU6(), "ReLU": torch.nn.ReLU(), "Swish": mb.Swish()}[act]
    h = (torch.randn(N, C, H, H, device=dev) * 1.5 + 0.3).to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last)
    h1 = h.clone().requires_grad_(True)
    h2 = h.float().clone().requires_grad_(True)
    y = engine.bn_act_apply(bn, actm, h1)
    y_ref = actm(ref(h2))
    assert _rel(y, y_ref) < 4e-3
    dy = torch.randn_like(y_ref)
    y.backward(dy.to(torch.bfloat16))
    y_ref.backward(dy.to(torch.bfloat16).float())
    assert _rel(h1.grad, h2.grad) < 1.5e-2
    assert _rel(bn.weight.grad, ref.weight.grad) < 1.5e-2
    assert _rel(bn.bias.grad, ref.bias.grad) < 1.5e-2
    if train:
        assert _rel(bn.running_mean, ref.running_mean) < 2e-3
        assert _rel(bn.running_var, ref.running_var) < 2e-3
        assert int(bn.num_batches_tracked) == int(ref.num_batches_tracked)
