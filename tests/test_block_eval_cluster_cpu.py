"""The small-batch cluster split of the one-launch eval block (csrc/block_eval.cuh, CLUSTER):
engine.eval_cluster_size on every single-branch block of the four configurations, the C ABI's
argument checks without a device, and the ptxas report of the cluster instantiations.  No GPU."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

from yet_another_mobilenet_series_b200 import engine
from yet_another_mobilenet_series_b200 import mobilenet_base as mb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMS = 132   # H100 SXM
BATCHES = (1, 8, 64, 256)

# cluster size per block (one entry per N of BATCHES); None: a multi-branch block (not on this path)
WANT = {
    "mobilenet_v2": [(1, 1, 1, 1)] * 7 + [
        (4, 4, 1, 1), (4, 4, 1, 1), (4, 4, 1, 1), (4, 4, 1, 1), (8, 8, 1, 1), (8, 8, 1, 1),
        (8, 8, 2, 1), (8, 8, 4, 1), (8, 8, 4, 1), (8, 8, 2, 1)],
    "proxyless_mobile": [(1, 1, 1, 1)] * 7 + [
        (4, 2, 1, 1), (4, 4, 1, 1), (4, 4, 1, 1), (4, 4, 1, 1), (8, 8, 1, 1), (4, 4, 1, 1),
        (4, 4, 1, 1), (4, 4, 1, 1), (8, 8, 1, 1), (8, 8, 2, 1), (8, 8, 2, 1), (8, 8, 2, 1),
        (8, 8, 2, 1)],
    "autonl_l": [(1, 1, 1, 1)] * 8 + [
        (4, 2, 1, 1), (4, 4, 1, 1), (4, 4, 1, 1), (4, 4, 1, 1), (8, 8, 1, 1), (4, 4, 1, 1),
        (4, 4, 1, 1), (4, 4, 1, 1), (8, 8, 1, 1), (8, 8, 2, 1), (8, 8, 2, 1), (8, 8, 2, 1),
        (8, 8, 2, 1)],
    "atomnas_c+": [(1, 1, 1, 1)] + [None] * 21,
}


def _blocks(name):
    """(block, input height) of every inverted-residual block at the 224 input (stem stride 2)."""
    import bench
    from _cfg import build_from_cfg
    model = bench.build_model() if name == "mobilenet_v2" else build_from_cfg(name)[0]
    res, out = 112, []
    for m in model.modules():
        if isinstance(m, (mb.InvertedResidualChannels, mb.InvertedResidualChannelsFused)):
            out.append((m, res))
            res = (res - 1) // m.stride + 1
    return out


@pytest.mark.parametrize("name", sorted(WANT))
def test_cluster_size_rule(name):
    got = []
    for blk, h in _blocks(name):
        if len(blk.channels) != 1:
            got.append(None)
            continue
        ho = (h - 1) // blk.stride + 1
        got.append(tuple(engine.eval_cluster_size(blk.kernel_sizes[0], blk.stride, n, ho, ho,
                                                  blk.channels[0], blk.output_dim, SMS)
                         for n in BATCHES))
    assert got == WANT[name]
    # the benchmark's batch keeps the unsplit launch everywhere
    assert all(g is None or g[-1] == 1 for g in got)


def test_cluster_size_rule_limits():
    # no split below 4 slices of 64 hidden channels; S never exceeds the slices
    assert engine.eval_cluster_size(3, 1, 1, 7, 7, 64, 64, SMS) == 1
    assert engine.eval_cluster_size(3, 1, 1, 7, 7, 192, 64, SMS) == 1    # 3 slices
    assert engine.eval_cluster_size(3, 1, 1, 7, 7, 200, 64, SMS) == 4    # 4, the last partial
    assert engine.eval_cluster_size(3, 1, 1, 7, 7, 448, 64, SMS) == 4    # 7 slices
    assert engine.eval_cluster_size(3, 1, 1, 7, 7, 512, 64, SMS) == 8
    assert engine.eval_cluster_size(3, 1, 1, 7, 7, 256, 64, SMS) == 4
    # tiles * S <= SM count
    assert engine.eval_cluster_size(3, 1, 1, 7, 7, 960, 160, 8) == 8
    assert engine.eval_cluster_size(3, 1, 1, 7, 7, 960, 160, 7) == 4
    assert engine.eval_cluster_size(3, 1, 1, 7, 7, 960, 160, 1) == 1
    # the tile plan: two 7x7 images per tile below 161 output channels, one above
    assert engine.eval_tiles(3, 1, 5, 7, 7, 160) == 3
    assert engine.eval_tiles(3, 1, 5, 7, 7, 320) == 5
    assert engine.eval_tiles(3, 1, 1, 28, 28, 32) == 8      # 7x16 tiles
    assert engine.eval_tiles(3, 1, 1, 56, 56, 24) == 32     # 7x16 tiles (two 7x7 images: 64)
    assert engine.eval_tiles(5, 2, 1, 56, 56, 32) == 80     # k5 stride 2: 6x7 outputs
    assert engine.eval_tiles(7, 2, 1, 28, 28, 40) == 28     # k7 stride 2: 4x7 outputs


def test_cluster_override_default():
    assert engine.EVAL_CLUSTER is None


def _args():
    from yet_another_mobilenet_series_b200 import native as nat
    a = nat.BlockEval()
    a.N, a.H, a.W, a.Cin, a.Chid, a.Cout = 1, 8, 8, 16, 128, 16
    a.kernel, a.stride, a.act = 3, 1, 1
    return a


def test_cluster_abi_without_device(built_lib):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = built_lib
    a = _args()
    for fn in (lib.yamb_block_eval_cluster_fwd, lib.yamb_block_eval_cluster_pool_fwd):
        for bad in (0, 1, 3, 16, -2):
            assert fn(C.byref(a), bad, None) == -1, bad
            assert b"cluster size" in lib.yamb_last_error()
        for cs in (2, 4, 8):
            assert fn(C.byref(a), cs, None) == -2     # YAMB_ENODEV
        assert fn(None, 2, None) == -1


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    nvcc = os.environ.get("NVCC")
    if not (nvcc and os.path.exists(nvcc)):
        nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else \
            shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "yet_another_mobilenet_series_b200", "csrc", "block_eval_cluster.cu")
    out = str(tmp_path_factory.mktemp("ptxas") / "block_eval_cluster.o")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xptxas", "-v", "-c", src, "-o", out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout + r.stderr


def test_cluster_instantiations_match_the_tile_plan_and_spill_nothing(ptxas_report):
    """One cluster kernel per (tile geometry, expansion) pair the launcher names (parsed out of the
    header, tests/block_eval_cases.py) x (lean, generic activation) x (plain, gate, pool), and none
    of them spills."""
    import block_eval_cases as bc
    kernels, cur = {}, None
    for line in ptxas_report.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1) if "block_eval_kernel" in m.group(1) else None
            if cur:
                kernels[cur] = []
            continue
        if cur:
            kernels[cur].append(line)
    assert all(name.endswith("Lb1EEEv14CUtensorMap_stS3_S3_NS_12BlockEvalDevE") for name in kernels)
    # block_eval_kernel<EvGeom<K, S, TOH, TOW, TI, CPT>, EXPAND, LEAN, MODE, CLUSTER = true>
    pat = re.compile(r"EvGeomILi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)EEELb([01])ELb([01])"
                     r"ELi(\d)ELb1E")
    got = set()
    for name in kernels:
        m = pat.search(name)
        assert m, name
        v = tuple(int(g) for g in m.groups())
        got.add((bc.Geom(*v[:6]), bool(v[6]), bool(v[7]), v[8]))
    want = {(g, ex, lean, mode) for g, ex in bc.compiled_instantiations()
            for lean in (False, True) for mode in (0, 1, 2)}
    assert got == want, (sorted(got - want), sorted(want - got))
    # 14 (tile geometry, expansion) pairs x (lean, generic activation) x (plain, gate, pool)
    assert len(kernels) == len(want) == 84, sorted(kernels)
    for name, lines in kernels.items():
        props = " ".join(lines)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", props)
        assert m, (name, props)
        assert m.group(1) == "0" and m.group(2) == "0", (name, props)
