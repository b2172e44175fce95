"""Parameter gradients of every autograd Function on the sm_90a path, in both hand-over modes.

Autograd mode (no flat arena): each backward returns its gradients to autograd, which accumulates
them into `.grad`.  Direct mode (every parameter in a fused optimizer's flat arena): the kernels
accumulate straight into the arena views and autograd gets nothing.  A block whose parameters are
only partly in an arena falls back to autograd mode.  The kernels are deterministic (DESIGN.md §c),
so every comparison here is bitwise.
"""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

BN = {"momentum": 0.01, "eps": 1e-3}


def _mb():
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    return mb


def _act(name):
    return _mb().get_active_fn(name)


def _ir_one_branch():
    return _mb().InvertedResidualChannels(16, 16, 1, [48], [3], True, _act("nn.ReLU6"), BN), \
        (4, 16, 10, 10)


def _ir_two_branches():
    return _mb().InvertedResidualChannels(16, 16, 1, [48, 32], [3, 5], True, _act("nn.ReLU6"),
                                          BN), (4, 16, 10, 10)


def _ir_no_expand():
    return _mb().InvertedResidualChannels(16, 24, 1, [16], [3], False, _act("nn.ReLU"), BN), \
        (4, 16, 10, 10)


def _fused_se_nl(norm):
    def make():
        mb = _mb()
        blk = mb.InvertedResidualChannelsFused(24, 24, 1, [72], [3], True, _act("nn.Swish"), BN,
                                               se_ratio=0.25, nl_c=0.25, nl_s=1)
        blk.nl_op.bn = mb.get_nl_norm_fn(norm)(24, **BN)
        return blk, (2, 24, 12, 12)
    return make


def _atomnas_padded():
    return _mb().InvertedResidualChannelsFused(24, 24, 1, [15, 23, 13], [3, 5, 7], True,
                                               _act("nn.Swish"), BN, se_ratio=0.5), (2, 24, 12, 12)


def _head_pw():
    return _mb().ConvBNReLU(32, 64, kernel_size=1, active_fn=_act("nn.ReLU6"),
                            batch_norm_kwargs=BN), (4, 32, 7, 7)


def _stem():
    return _mb().ConvBNReLU(3, 16, kernel_size=3, stride=2, active_fn=_act("nn.ReLU6"),
                            batch_norm_kwargs=BN), (4, 3, 32, 32)


def _torch_conv():
    # a convolution neither the stem nor the pointwise kernels take: torch runs it, the
    # BatchNorm + activation behind it run on engine.bn_act_apply
    return _mb().ConvBNReLU(16, 32, kernel_size=3, active_fn=_act("nn.ReLU"),
                            batch_norm_kwargs=BN), (4, 16, 8, 8)


def _classifier():
    return torch.nn.Sequential(torch.nn.Linear(64, 16)), (8, 64)


CASES = {
    "ir_one_branch": _ir_one_branch,
    "ir_two_branches": _ir_two_branches,
    "ir_no_expand": _ir_no_expand,
    "fused_se_nl_batchnorm": _fused_se_nl("nn.BatchNorm"),
    "fused_se_nl_instancenorm": _fused_se_nl("nn.InstanceNorm"),
    "atomnas_padded": _atomnas_padded,
    "head_pw_conv": _head_pw,
    "stem": _stem,
    "torch_conv_bn_act": _torch_conv,
    "classifier": _classifier,
}


def _forward(mod, x):
    if isinstance(mod, torch.nn.Sequential) and isinstance(mod[0], torch.nn.Linear):
        from yet_another_mobilenet_series_b200 import mobilenet_supernet as sup
        return sup.run_classifier(mod, x)
    return mod(x)


@pytest.fixture
def deterministic_cudnn():
    """The torch-run convolution's own gradients come from cuDNN: pin its algorithms."""
    saved = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = saved


class _Case:
    """A seeded module (copied fresh for every mode) and two seeded batches A, B."""

    def __init__(self, name):
        torch.manual_seed(7)
        base, shape = CASES[name]()
        base.apply(_mb().init_weights_mnas)
        for m in base.modules():
            if isinstance(m, (torch.nn.BatchNorm2d, torch.nn.InstanceNorm2d)) and m.affine:
                m.weight.data.uniform_(0.5, 1.5)       # ZeroInitBN would switch a branch off
                m.bias.data.normal_(0.0, 0.1)
        self.base = base.cuda().train()
        gen = torch.Generator().manual_seed(11)
        self.x = [torch.randn(shape, generator=gen).mul_(0.5).cuda() for _ in range(2)]
        with torch.no_grad():
            yshape = _forward(copy.deepcopy(self.base), self.x[0]).shape
        self.dy = [torch.randn(yshape, generator=gen).cuda() for _ in range(2)]

    def fresh(self):
        return copy.deepcopy(self.base)

    def backward(self, mod, b=0):
        y = _forward(mod, self.x[b])
        y.backward(self.dy[b].to(y.dtype))
        torch.cuda.synchronize()

    def autograd_grads(self):
        """Gradients of batch A from a module without an arena (autograd mode)."""
        mod = self.fresh()
        self.backward(mod)
        return [p.grad.clone() for p in mod.parameters()]


def _names(mod):
    return [n for n, _ in mod.named_parameters()]


def _assert_equal(got, want, mod, what):
    for n, g, w in zip(_names(mod), got, want):
        assert g is not None, (what, n)
        assert torch.equal(g, w), (what, n, float((g - w).abs().max()))


@pytest.mark.parametrize("name", list(CASES))
def test_autograd_mode_accumulates(built_lib, deterministic_cudnn, name):
    case = _Case(name)
    mod = case.fresh()
    case.backward(mod)
    first = [p.grad.clone() for p in mod.parameters()]
    assert all(bool(g.abs().sum() > 0) for g in first), name
    case.backward(mod)
    _assert_equal([p.grad for p in mod.parameters()], [2 * g for g in first], mod, "twice")


@pytest.mark.parametrize("name", list(CASES))
def test_returned_gradients_are_not_aliased(built_lib, deterministic_cudnn, name):
    case = _Case(name)
    mod = case.fresh()
    params = list(mod.parameters())
    y = _forward(mod, case.x[0])
    got = torch.autograd.grad(y, params, case.dy[0].to(y.dtype))
    kept = [g.clone() for g in got]
    case.backward(mod, 1)
    _assert_equal(got, kept, mod, "batch A after batch B")
    _assert_equal(kept, case.autograd_grads(), mod, "autograd.grad vs backward")


@pytest.mark.parametrize("name", list(CASES))
def test_direct_mode_equals_autograd_mode(built_lib, deterministic_cudnn, name):
    from yet_another_mobilenet_series_b200.fused_rmsprop import RMSprop
    case = _Case(name)
    want = case.autograd_grads()
    mod = case.fresh()
    opt = RMSprop(mod.parameters(), lr=0.01, momentum=0.9)
    A = opt.arenas()
    assert float(A["g"].abs().sum()) == 0.0
    ptrs = [p.grad.data_ptr() for p in mod.parameters()]
    case.backward(mod)
    assert [p.grad.data_ptr() for p in mod.parameters()] == ptrs
    _assert_equal([p.grad for p in mod.parameters()], want, mod, "direct vs autograd")
    case.backward(mod)
    assert [p.grad.data_ptr() for p in mod.parameters()] == ptrs
    _assert_equal([p.grad for p in mod.parameters()], [2 * g for g in want], mod, "direct twice")


@pytest.mark.parametrize("name", list(CASES))
def test_mixed_ownership_falls_back_to_autograd(built_lib, deterministic_cudnn, name):
    from yet_another_mobilenet_series_b200.fused_rmsprop import RMSprop
    case = _Case(name)
    want = case.autograd_grads()
    mod = case.fresh()
    params = list(mod.parameters())
    opt = RMSprop(params[::2], lr=0.01, momentum=0.9)
    opt.arenas()
    case.backward(mod)
    _assert_equal([p.grad for p in params], want, mod, "mixed ownership")
