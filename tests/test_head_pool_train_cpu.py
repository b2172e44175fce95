"""CPU: the dispatch rule of the training-mode head (tail_ops.head_pool_train_covered, with the
full-extent pool check of run_features), the ABI struct sizes of yamb_head_pool_train{,_grad},
and the entry points' answers without a device."""
import ctypes as C
import types

import pytest
import torch


def _head(Cin=320, Cout=1280, act="nn.ReLU6"):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    return mb.ConvBNReLU(Cin, Cout, kernel_size=1, active_fn=mb.get_active_fn(act))


def _x(N=4, C=320, hw=7):
    """What the rule reads of a CUDA activation (a CPU test has none)."""
    return types.SimpleNamespace(is_cuda=True, shape=(N, C, hw, hw))


@pytest.fixture
def switch(monkeypatch):
    from yet_another_mobilenet_series_b200 import engine
    monkeypatch.setattr(engine, "TRAIN_TAIL_FUSED", True)
    return engine


def test_covered_in_training_with_the_switch_on(switch):
    from yet_another_mobilenet_series_b200 import tail_ops
    for act in ("nn.ReLU", "nn.ReLU6", "nn.Swish", "nn.HSwish"):
        assert tail_ops.head_pool_train_covered(_head(act=act).train(), _x())


def test_switch_off_by_default():
    from yet_another_mobilenet_series_b200 import engine, tail_ops
    assert engine.TRAIN_TAIL_FUSED is False
    assert not tail_ops.head_pool_train_covered(_head().train(), _x())


def test_eval_mode_and_running_statistics_take_the_unfused_path(switch):
    from yet_another_mobilenet_series_b200 import tail_ops
    assert not tail_ops.head_pool_train_covered(_head().eval(), _x())
    # a BatchNorm without running statistics normalises with batch statistics even in eval()
    h = _head()
    h[1] = torch.nn.BatchNorm2d(1280, track_running_stats=False)
    assert tail_ops.head_pool_train_covered(h.eval(), _x())


@pytest.mark.parametrize("cin,cout", [(320, 1276), (324, 1280)])
def test_channels_not_multiple_of_8(switch, cin, cout):
    from yet_another_mobilenet_series_b200 import tail_ops
    assert not tail_ops.head_pool_train_covered(_head(cin, cout).train(), _x(C=cin))


def test_cpu_tensor_and_other_convolutions(switch):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    from yet_another_mobilenet_series_b200 import tail_ops
    assert not tail_ops.head_pool_train_covered(_head().train(), torch.zeros(2, 320, 7, 7))
    conv3 = mb.ConvBNReLU(320, 1280, kernel_size=3, active_fn=mb.get_active_fn("nn.ReLU6"))
    assert not tail_ops.head_pool_train_covered(conv3.train(), _x())
    assert tail_ops.head_pool_train(_head().eval(), _x()) is None


def test_only_a_full_extent_pool_is_fused():
    from yet_another_mobilenet_series_b200.mobilenet_supernet import _full_extent
    x = torch.zeros(2, 1280, 7, 7)
    assert _full_extent(torch.nn.AvgPool2d(7), x)
    assert not _full_extent(torch.nn.AvgPool2d(3), x)
    assert not _full_extent(torch.nn.AvgPool2d(7, stride=1), x)
    assert not _full_extent(torch.nn.AvgPool2d(7, padding=1), torch.zeros(2, 1280, 7, 7))


def test_struct_sizes(built_lib):
    from yet_another_mobilenet_series_b200 import native as nat
    assert built_lib.yamb_struct_size(31) == C.sizeof(nat.HeadPoolTrain)
    assert built_lib.yamb_struct_size(32) == C.sizeof(nat.HeadPoolTrainGrad)
    for name in ("yamb_head_pool_train_fwd", "yamb_head_pool_train_bwd"):
        assert name in nat.SYMBOLS and hasattr(built_lib, name)


def _args(nat, **kw):
    a, g = nat.HeadPoolTrain(), nat.HeadPoolTrainGrad()
    for s in (a, g):
        s.N, s.HW, s.C, s.act = 4, 49, 1280, 2
        s.h, s.scale, s.shift = 4096, 8192, 12288       # aligned stand-ins, never dereferenced
    a.pooled = 16384
    g.dpooled, g.dh = 16384, 20480
    b = g.bn
    b.partials, b.counter, b.mean, b.invstd = 24576, 28672, 32768, 36864
    b.ca, b.cb, b.cc, b.count = 40960, 45056, 49152, 4 * 49
    for s in (a, g):
        for k, v in kw.items():
            setattr(s, k, v)
    return a, g


def test_no_device_and_refused_arguments(built_lib):
    """Valid arguments without a device: YAMB_ENODEV; arguments the kernels do not cover:
    YAMB_EINVAL, with or without a device.  Nothing is dereferenced either way."""
    from yet_another_mobilenet_series_b200 import native as nat
    if torch.cuda.is_available():
        pytest.skip("checks the answers without a device")
    a, g = _args(nat)
    assert built_lib.yamb_head_pool_train_fwd(C.byref(a), None) == -2
    assert built_lib.yamb_head_pool_train_bwd(C.byref(g), None) == -2
    for kw in ({"C": 1276}, {"C": 0}, {"N": 0}, {"HW": 0}, {"act": 5}, {"h": 4098},
               {"scale": None}):
        a, g = _args(nat, **kw)
        assert built_lib.yamb_head_pool_train_fwd(C.byref(a), None) == -1, kw
        assert built_lib.yamb_head_pool_train_bwd(C.byref(g), None) == -1, kw
    a, g = _args(nat)
    a.pooled = None
    assert built_lib.yamb_head_pool_train_fwd(C.byref(a), None) == -1
    g.bn.count = 4 * 49 + 1
    assert built_lib.yamb_head_pool_train_bwd(C.byref(g), None) == -1
    _, g = _args(nat)
    g.dpooled = None
    assert built_lib.yamb_head_pool_train_bwd(C.byref(g), None) == -1
    assert built_lib.yamb_head_pool_train_fwd(None, None) == -1
