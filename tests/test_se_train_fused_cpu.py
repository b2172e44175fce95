"""CPU: the training-mode Squeeze-and-Excitation backward (TrainStep(fused_se=True)): which blocks
of the SE configurations take it, the ABI struct sizes of the three new entry points, their answers
without a device and to refused arguments, the ptxas report of every new depthwise instantiation,
and that the existing depthwise backward kernels compile to the SASS they compiled to before."""
import ctypes as C
import hashlib
import json
import os
import re
import subprocess
import sys
import types

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "yet_another_mobilenet_series_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17"]


@pytest.fixture
def flags(monkeypatch):
    """A stand-in for the reference's utils.config (the non-local block reads FLAGS)."""
    mod = types.ModuleType("utils.config")
    mod.FLAGS = types.SimpleNamespace()
    monkeypatch.setitem(sys.modules, "utils.config", mod)
    return mod


def test_switch_off_by_default():
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    import inspect
    assert engine.TRAIN_SE_FUSED is False
    assert inspect.signature(TrainStep).parameters["fused_se"].default is False


def _blocks(model):
    from yet_another_mobilenet_series_b200 import engine
    return [m for m in model.features if hasattr(m, "expand_conv") or hasattr(m, "ops")
            if engine.block_parts(m) is not None]


def _model(name):
    """The "+" configurations: atomnas_a+ / b+ from the multi-branch fixture, the others from
    tests/golden/model_cfgs.json (AutoNL-S is in neither)."""
    from _cfg import build_from_cfg
    if name in ("atomnas_a+", "atomnas_b+"):
        from test_block_eval_mb_cpu import build
        return build(name)
    return build_from_cfg(name)[0]


@pytest.mark.parametrize("name", ["atomnas_a+", "atomnas_b+", "atomnas_c+", "autonl_l"])
def test_routing(flags, monkeypatch, name):
    """With the switch on, every block with SE takes the path (multi-branch blocks, the
    non-expanding block 1 and the SE + non-local blocks included) and no other block does; with it
    off, none does.  BlockPlan.backward decides through the same predicate (engine._se_fused)."""
    import inspect
    from yet_another_mobilenet_series_b200 import engine
    assert "_se_fused(self.se)" in inspect.getsource(engine.BlockPlan.backward)
    model = _model(name)
    blocks = _blocks(model)
    se = [engine.block_parts(b).se is not None for b in blocks]
    assert sum(se) > 0
    assert not any(engine.se_backward_fused(b) for b in blocks)
    monkeypatch.setattr(engine, "TRAIN_SE_FUSED", True)
    assert [engine.se_backward_fused(b) for b in blocks] == se
    kinds = {(len(b.channels) > 1, bool(b.expand), engine.block_parts(b).nl is not None)
             for b, s in zip(blocks, se) if s}
    if name.startswith("atomnas"):
        assert any(k[0] for k in kinds), kinds          # multi-branch SE blocks
        assert any(not k[1] for k in kinds), kinds      # block 1: SE without expansion
    else:
        assert any(k[2] for k in kinds), kinds          # SE + non-local


def test_struct_sizes(built_lib):
    from yet_another_mobilenet_series_b200 import native as nat
    assert built_lib.yamb_struct_size(37) == C.sizeof(nat.SeBwdStats)
    assert built_lib.yamb_struct_size(38) == C.sizeof(nat.SeBnBwdFinalize)
    assert built_lib.yamb_struct_size(39) == C.sizeof(nat.DwBwdSe)
    for fn in ("yamb_se_bwd_stats_bwd", "yamb_se_bn_bwd_finalize", "yamb_depthwise_bwd_se"):
        assert fn in nat.SYMBOLS and hasattr(built_lib, fn)


def _stats(nat, **kw):
    a = nat.SeBwdStats()
    a.N, a.HW, a.C, a.ldd, a.ldh, a.act = 4, 49, 144, 144, 144, 2
    a.dy, a.h, a.scale, a.shift, a.mean, a.invstd = 4096, 8192, 12288, 16384, 20480, 24576
    a.dgate, a.sums = 28672, 32768
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _finalize(nat, **kw):
    bn = nat.BnBwd()
    bn.mean, bn.invstd, bn.ca, bn.cb, bn.cc, bn.count = 4096, 8192, 12288, 16384, 20480, 196
    f = nat.SeBnBwdFinalize()
    f.N, f.C, f.lds, f.ldg = 4, 48, 144, 144
    f.sums, f.gate, f.dpool, f.bn = 24576, 28672, 32768, C.pointer(bn)
    for k, v in kw.items():
        if k.startswith("bn_"):
            setattr(bn, k[3:], v)
        else:
            setattr(f, k, v)
    return f, bn


def _dwse(nat, **kw):
    a = nat.DwBwdSe()
    d = a.dw
    d.N, d.H, d.W, d.C, d.ldc, d.k, d.stride = 2, 14, 14, 48, 144, 3, 1
    d.dz, d.h, d.ca, d.cb, d.cc, d.w, d.dw, d.x, d.dx = (4096 * i for i in range(1, 10))
    a.gate, a.dpool, a.ldg, a.scale, a.shift, a.act = 40960, 45056, 144, 49152, 53248, 2
    for k, v in kw.items():
        if k.startswith("dw_"):
            setattr(a.dw, k[3:], v)
        else:
            setattr(a, k, v)
    return a


def test_no_device(built_lib):
    """Valid arguments without a device: YAMB_ENODEV."""
    import torch
    from yet_another_mobilenet_series_b200 import native as nat
    if torch.cuda.is_available():
        pytest.skip("checks the answers without a device")
    lib = built_lib
    assert lib.yamb_se_bwd_stats_bwd(C.byref(_stats(nat)), None) == -2
    f, _bn = _finalize(nat)
    assert lib.yamb_se_bn_bwd_finalize(C.byref(f), None) == -2
    for k, s in ((3, 1), (5, 2), (7, 1)):
        for c in (8, 16, 48, 96, 144):
            a = _dwse(nat, dw_k=k, dw_stride=s, dw_C=c, dw_H=56, dw_W=56)
            assert lib.yamb_depthwise_bwd_se(C.byref(a), None) == -2, (k, s, c)


def test_refused_arguments(built_lib):
    """Malformed arguments: YAMB_EINVAL, with or without a device.  Every one of these checks comes
    before the device query (the no-device test shows the same arguments reach it otherwise), so
    the stand-in pointers are never used."""
    from yet_another_mobilenet_series_b200 import native as nat
    lib = built_lib
    for kw in ({"N": 0}, {"HW": 0}, {"C": 0}, {"C": 12}, {"N": 65536}, {"ldd": 100}, {"ldh": 140},
               {"dy": None}, {"h": 8200}, {"scale": None}, {"mean": None}, {"invstd": None},
               {"dgate": None}, {"sums": None}, {"act": 5}, {"act": -1}):
        assert lib.yamb_se_bwd_stats_bwd(C.byref(_stats(nat, **kw)), None) == -1, kw
    for kw in ({"N": 0}, {"C": 0}, {"lds": 40}, {"ldg": 40}, {"sums": None}, {"gate": None},
               {"dpool": None}, {"bn_mean": None}, {"bn_ca": None}, {"bn_cc": None},
               {"bn_count": 0}):
        f, _bn = _finalize(nat, **kw)
        assert lib.yamb_se_bn_bwd_finalize(C.byref(f), None) == -1, kw
    f, _bn = _finalize(nat)
    f.bn = None
    assert lib.yamb_se_bn_bwd_finalize(C.byref(f), None) == -1
    for kw in ({"gate": None}, {"dpool": None}, {"scale": None}, {"shift": None},
               {"gate": 40968}, {"dpool": 45060}, {"scale": 49156}, {"ldg": 40}, {"ldg": 146},
               {"act": 7}, {"dw_k": 4}, {"dw_stride": 3}, {"dw_C": 12}, {"dw_N": 0},
               {"dw_dz": None}, {"dw_dz": 4104}, {"dw_dx": 4100}, {"dw_ca": None}):
        assert lib.yamb_depthwise_bwd_se(C.byref(_dwse(nat, **kw)), None) == -1, kw
    for fn in (lib.yamb_se_bwd_stats_bwd, lib.yamb_se_bn_bwd_finalize, lib.yamb_depthwise_bwd_se):
        assert fn(None, None) == -1


def _ptxas(tmp_path, name):
    src = os.path.join(CSRC, name + ".cu")
    out = subprocess.run([NVCC] + FLAGS + ["-cubin", "-Xptxas", "-v", "-o",
                                           str(tmp_path / (name + ".cubin")), src],
                         capture_output=True, text=True, check=True).stderr
    rows = re.findall(r"Function properties for (\w+)\n\s*\d+ bytes stack frame, (\d+) bytes "
                      r"spill stores, (\d+) bytes spill loads\nptxas info\s*: Used (\d+) registers",
                      out)
    return {k: (int(s), int(l), int(r)) for k, s, l, r in rows}


def _inst(name):
    m = re.search(r"dw_bwd(?:_se)?_kernelILi(\d)ELi(\d)ELi(\d+)ELi(\d+)ELi(\d+)ELb(\d)", name)
    return tuple(int(g) for g in m.groups())


@pytest.mark.skipif(not os.path.exists(NVCC), reason="no nvcc")
def test_new_instantiations_ptxas(tmp_path):
    """Every (k, stride, channel tile, tap split, DGRAD) of yamb_depthwise_bwd is built for the SE
    variant too, within the register cap of __launch_bounds__ (k = 3: kDw3MinBlocks CTAs per SM),
    spilling no more than the dw_bwd kernel of the same instantiation plus 64 bytes.  (The 3x3
    dw_bwd kernels themselves spill at their 128-register cap.)"""
    min_blocks = int(re.search(r"kDw3MinBlocks = (\d+)",
                               open(os.path.join(CSRC, "depthwise.cuh")).read()).group(1))
    base, se = {}, {}
    for f, dst in (("depthwise", base), ("depthwise_narrow", base), ("depthwise_se", se),
                   ("depthwise_se_narrow", se)):
        for k, v in _ptxas(tmp_path, f).items():
            if "dw_bwd_kernel" in k or "dw_bwd_se_kernel" in k:
                dst[_inst(k)] = v
    assert len(base) == 32 and set(se) == set(base), sorted(set(base) ^ set(se))
    report = []
    for inst, (st, ld, regs) in sorted(se.items()):
        bst, bld, _ = base[inst]
        report.append("%s se %d/%d B spilled, %d regs; dw_bwd %d/%d" % (inst, st, ld, regs, bst, bld))
        assert regs <= (65536 // (256 * min_blocks) if inst[0] == 3 else 255), report[-1]
        assert st <= bst + 64 and ld <= bld + 64, "\n".join(report)


def _sass_digests(obj):
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", obj], capture_output=True,
                         text=True, check=True).stdout
    digests, cur, body = {}, None, []
    for line in out.splitlines() + ["Function : <end>"]:
        m = re.search(r"Function : (\S+)", line)
        if m:
            if cur and "dw_bwd_kernel" in cur:
                digests[cur] = hashlib.sha256("\n".join(body).encode()).hexdigest()
            cur, body = m.group(1), []
        elif cur and line.strip():
            body.append(line.rstrip())
    return digests


@pytest.mark.skipif(not os.path.exists(NVCC), reason="no nvcc")
def test_existing_dw_bwd_sass_unchanged(tmp_path):
    """The dw_bwd kernels compile to the instructions they compiled to before the SE variant shared
    their source (tests/golden/dw_bwd_sass.json: SHA-256 of each kernel's cuobjdump -sass text, from
    the build of the parent commit with CUDA 12.9)."""
    with open(os.path.join(ROOT, "tests", "golden", "dw_bwd_sass.json")) as f:
        golden = json.load(f)
    ver = subprocess.run([NVCC, "--version"], capture_output=True, text=True).stdout
    if golden["nvcc"] not in ver:
        pytest.skip("SASS digests are from nvcc %s" % golden["nvcc"])
    got = {}
    for name in ("depthwise", "depthwise_narrow"):
        obj = str(tmp_path / (name + ".o"))
        subprocess.run([NVCC] + FLAGS + ["-lineinfo", "-Xcompiler", "-fPIC", "-c",
                                         os.path.join(CSRC, name + ".cu"), "-o", obj], check=True)
        got.update(_sass_digests(obj))
    assert len(golden["kernels"]) == 32
    assert got == golden["kernels"]
