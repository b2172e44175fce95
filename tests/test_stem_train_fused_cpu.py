"""CPU: the coverage rule of the training-mode stem + first block (tail_ops.stem_block_fused_covered)
on the four configurations and on the cases it declines, the ABI struct sizes of
yamb_stem_conv_train{,_grad}, the entry points' answers without a device, and the new kernels'
spill-free compile for sm_90a."""
import ctypes as C
import os
import re
import subprocess
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def flags(monkeypatch):
    """A stand-in for the reference's utils.config (the non-local block reads FLAGS)."""
    mod = types.ModuleType("utils.config")
    mod.FLAGS = types.SimpleNamespace()
    monkeypatch.setitem(sys.modules, "utils.config", mod)
    return mod


def _x(N=8, hw=224):
    """What the rule reads of a CUDA image batch (a CPU test has none)."""
    return types.SimpleNamespace(is_cuda=True, shape=(N, 3, hw, hw))


@pytest.mark.parametrize("name", ["mobilenet_v2", "proxyless_mobile", "atomnas_c+", "autonl_l"])
def test_covered_on_every_configuration(flags, name):
    from _cfg import build_from_cfg
    from yet_another_mobilenet_series_b200 import tail_ops
    model, cfg = build_from_cfg(name)
    model.train()
    stem, block = model.features[0], model.features[1]
    assert tail_ops.stem_block_fused_covered(stem, block, _x(hw=cfg["flags"]["image_size"]))
    assert not tail_ops.stem_block_fused_covered(stem, block, torch.zeros(2, 3, 32, 32))  # CPU x
    model.eval()
    assert not tail_ops.stem_block_fused_covered(stem, block, _x())      # eval-mode BatchNorm


def _pair(t=1, c=16, s=1, cin=32, stem_c=32, act="nn.ReLU6", ks=(3,)):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    from yet_another_mobilenet_series_b200.mobilenet_supernet import get_block_wrapper
    a = mb.get_active_fn(act)
    stem = mb.ConvBNReLU(3, stem_c, stride=2, active_fn=a)
    block = get_block_wrapper("InvertedResidualChannels")(cin, c, s, t, list(ks), active_fn=a)
    return stem.train(), block.train()


def test_declined_pairs():
    from yet_another_mobilenet_series_b200 import tail_ops
    assert tail_ops.stem_block_fused_covered(*_pair(), _x())
    assert tail_ops.stem_block_fused_covered(*_pair(act="nn.Swish"), _x())
    assert not tail_ops.stem_block_fused_covered(*_pair(t=6), _x())             # expansion
    assert not tail_ops.stem_block_fused_covered(*_pair(c=32), _x())            # skip connection
    assert not tail_ops.stem_block_fused_covered(*_pair(cin=24, stem_c=24), _x())   # stem caps
    stem, block = _pair()
    assert not tail_ops.stem_block_fused_covered(stem, torch.nn.Identity(), _x())
    stem.eval()
    assert not tail_ops.stem_block_fused_covered(stem, block, _x())          # running statistics
    stem[1] = torch.nn.BatchNorm2d(32, track_running_stats=False)
    assert tail_ops.stem_block_fused_covered(stem, block, _x())              # batch statistics
    stem, block = _pair()
    stem[0] = torch.nn.Conv2d(3, 32, 3, 1, 1, bias=False)                    # stride 1
    assert not tail_ops.stem_block_fused_covered(stem, block, _x())


def test_switch_off_by_default():
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    import inspect
    assert engine.TRAIN_STEM_FUSED is False
    assert inspect.signature(TrainStep).parameters["fused_stem"].default is False


def test_struct_sizes(built_lib):
    from yet_another_mobilenet_series_b200 import native as nat
    assert built_lib.yamb_struct_size(33) == C.sizeof(nat.StemConvTrain)
    assert built_lib.yamb_struct_size(34) == C.sizeof(nat.StemConvTrainGrad)
    for name in ("yamb_stem_conv_train_fwd", "yamb_stem_conv_train_wgrad"):
        assert name in nat.SYMBOLS and hasattr(built_lib, name)


def _args(nat, N=4, H=225, W=223, Cout=32, **kw):
    """Aligned stand-ins for every pointer; nothing is dereferenced without a device."""
    bn = nat.BnFwd()
    bn.partials, bn.counter, bn.scale, bn.shift = 4096, 8192, 12288, 16384
    bn.count = N * ((H - 1) // 2 + 1) * ((W - 1) // 2 + 1)
    a, g = nat.StemConvTrain(), nat.StemConvTrainGrad()
    for s in (a, g):
        s.N, s.H, s.W, s.Cout, s.x = N, H, W, Cout, 20480
        s.mean[:] = (0.485, 0.456, 0.406)
        s.std[:] = (0.229, 0.224, 0.225)
    a.w, a.y, a.bn = 24576, 28672, C.pointer(bn)
    g.dz, g.h, g.ca, g.cb, g.cc, g.dw = 32768, 36864, 40960, 45056, 49152, 53248
    for s in (a, g):
        for k, v in kw.items():
            if hasattr(s, k):
                setattr(s, k, v)
    return a, g, bn


def test_no_device_and_refused_arguments(built_lib):
    """Valid arguments without a device: YAMB_ENODEV; arguments outside the caps: YAMB_EINVAL,
    with or without a device."""
    from yet_another_mobilenet_series_b200 import native as nat
    if torch.cuda.is_available():
        pytest.skip("checks the answers without a device")
    for u8 in (0, 1):
        for cout in (8, 16, 32, 64):
            a, g, _bn = _args(nat, Cout=cout, x_u8=u8)
            assert built_lib.yamb_stem_conv_train_fwd(C.byref(a), None) == -2
            assert built_lib.yamb_stem_conv_train_wgrad(C.byref(g), None) == -2
    for kw in ({"Cout": 24}, {"Cout": 48}, {"Cout": 72}, {"Cout": 0}, {"N": 0}, {"H": 0},
               {"x": None}, {"x_u8": 2}):
        a, g, _bn = _args(nat, **kw)
        assert built_lib.yamb_stem_conv_train_fwd(C.byref(a), None) == -1, kw
        assert built_lib.yamb_stem_conv_train_wgrad(C.byref(g), None) == -1, kw
    for kw in ({"w": None}, {"y": None}, {"y": 28674}, {"bn": None}):
        a, _g, _bn = _args(nat, **kw)
        assert built_lib.yamb_stem_conv_train_fwd(C.byref(a), None) == -1, kw
    a, _g, bn = _args(nat)
    bn.count += 1
    assert built_lib.yamb_stem_conv_train_fwd(C.byref(a), None) == -1
    a, _g, bn = _args(nat)
    bn.partials = None
    assert built_lib.yamb_stem_conv_train_fwd(C.byref(a), None) == -1
    for kw in ({"dz": None}, {"h": None}, {"h": 36866}, {"dz": 32776}, {"ca": None},
               {"cc": None}, {"dw": None}):
        _a, g, _bn = _args(nat, **kw)
        assert built_lib.yamb_stem_conv_train_wgrad(C.byref(g), None) == -1, kw
    a, g, _bn = _args(nat, x_u8=1)
    a.std[1] = 0.0
    g.mean[0] = float("nan")
    assert built_lib.yamb_stem_conv_train_fwd(C.byref(a), None) == -1
    assert built_lib.yamb_stem_conv_train_wgrad(C.byref(g), None) == -1
    assert built_lib.yamb_stem_conv_train_fwd(None, None) == -1
    assert built_lib.yamb_stem_conv_train_wgrad(None, None) == -1


def test_new_kernels_compile_without_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    src = os.path.join(ROOT, "yet_another_mobilenet_series_b200", "csrc", "stem.cu")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                          "-cubin", "-Xptxas", "-v", "-o", str(tmp_path / "stem.cubin"), src],
                         capture_output=True, text=True, check=True).stderr
    props = re.findall(r"Function properties for (\w+)\n\s*\d+ bytes stack frame, (\d+) bytes "
                       r"spill stores, (\d+) bytes spill loads", out)
    train = {k: (int(s), int(l)) for k, s, l in props if "train_kernel" in k}
    assert len(train) == 4, train           # fwd / wgrad x bf16 / uint8
    assert all(v == (0, 0) for v in train.values()), train
