"""Small-batch eval of the searched networks (csrc/block_eval_mb_cluster.cu, engine.EVAL_SMALL_BATCH)
without a GPU: engine.eval_cluster_size on the packed multi-branch blocks of AtomNAS-C / C+, the
routing of the switch and SMALL_BATCH_FASTER, EvalStep setting the switch only around its eval
forwards, the C ABI's argument checks, and the ptxas report of the new instantiations."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

from test_block_eval_mb_cpu import MB_GEOMS
from test_block_eval_mb_cpu import build as build_mb
from yet_another_mobilenet_series_b200 import engine
from yet_another_mobilenet_series_b200 import mobilenet_base as mb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMS = 132   # H100 SXM
BATCHES = (1, 8, 64, 256)
NETWORKS = ("atomnas_c", "atomnas_c+", "autonl_l")

# cluster size of every multi-branch block of AtomNAS-C and C+ (the same packed shapes), one entry
# per N of BATCHES: 1 below 4 slices of 64 packed channels
WANT_ATOMNAS = [
    (1, 1, 1, 1), (1, 1, 1, 1), (1, 1, 1, 1), (1, 1, 1, 1), (4, 1, 1, 1), (1, 1, 1, 1),
    (1, 1, 1, 1), (1, 1, 1, 1), (8, 2, 1, 1), (1, 1, 1, 1), (1, 1, 1, 1), (1, 1, 1, 1),
    (8, 4, 1, 1), (1, 1, 1, 1), (1, 1, 1, 1), (1, 1, 1, 1), (8, 8, 1, 1), (8, 8, 2, 1),
    (8, 8, 2, 1), (8, 8, 2, 1), (8, 8, 2, 1)]


def _model(name):
    if name.startswith("atomnas"):
        return build_mb(name)
    from _cfg import build_from_cfg
    return build_from_cfg(name)[0]


def _blocks(model):
    """(block, input height) of every inverted-residual block at the 224 input (stem stride 2)."""
    res, out = 112, []
    for m in model.modules():
        if isinstance(m, (mb.InvertedResidualChannels, mb.InvertedResidualChannelsFused)):
            out.append((m, res))
            res = (res - 1) // m.stride + 1
    return out


@pytest.mark.parametrize("name", ["atomnas_c", "atomnas_c+"])
def test_cluster_size_on_packed_blocks(name):
    got = []
    for blk, h in _blocks(_model(name)):
        if len(blk.channels) == 1:
            continue
        lay = engine.mb_layout(blk.kernel_sizes, blk.channels)
        ho = (h - 1) // blk.stride + 1
        sizes = tuple(engine.eval_cluster_size(lay.kmax, blk.stride, n, ho, ho, lay.Chid,
                                               blk.output_dim, SMS) for n in BATCHES)
        nc = -(-lay.Chid // 64)
        for n, s in zip(BATCHES, sizes):
            tiles = engine.eval_tiles(lay.kmax, blk.stride, n, ho, ho, blk.output_dim)
            assert s == 1 or (nc >= 4 and s <= nc and tiles * s <= SMS), (lay.Chid, n, s)
        got.append(sizes)
    assert got == WANT_ATOMNAS


# ---- the switch --------------------------------------------------------------------------------
def test_defaults():
    assert engine.EVAL_SMALL_BATCH is False and engine.SMALL_BATCH_RULE is True
    assert isinstance(engine.SMALL_BATCH_FASTER, tuple)
    for kind, n in engine.SMALL_BATCH_FASTER:
        assert isinstance(n, int) and n >= 1, (kind, n)


def test_listed_kinds_exist_in_the_configs():
    """Every kind of SMALL_BATCH_FASTER is a multi-branch kind, or a fused-class kind the N = 256
    rule keeps off, of AtomNAS-C, C+ or AutoNL-L."""
    kinds = set()
    for name in NETWORKS:
        for blk, _ in _blocks(_model(name)):
            kind = engine.small_batch_kind(blk)
            if kind[0] == "mb" or (engine.block_parts(blk).fused and (kind[1] != 3 or not kind[3])):
                kinds.add(kind)
    for kind, _ in engine.SMALL_BATCH_FASTER:
        assert kind in kinds, kind


def _routes(model, n):
    x = torch.zeros(n, 8, 14, 14)
    out = []
    with torch.no_grad():
        for blk, _ in _blocks(model):
            out.append("one" if engine.eval_supported(blk, x) else
                       "mb" if engine.eval_mb_supported(blk, x) else "four")
    return out


@pytest.mark.parametrize("name", NETWORKS)
def test_routing(monkeypatch, name):
    """Off: the routes of the parent.  On with the rule off: every multi-branch block on the
    multi-branch path and every fused-class block on the one-launch path, at any N.  On with the
    rule: exactly the listed kinds up to their bound."""
    model = _model(name).eval()
    blocks = [b for b, _ in _blocks(model)]
    base = {n: _routes(model, n) for n in (1, 256)}
    monkeypatch.setattr(engine, "EVAL_SMALL_BATCH", True)
    monkeypatch.setattr(engine, "SMALL_BATCH_RULE", False)
    for n in (1, 256):
        got = _routes(model, n)
        for b, r0, r in zip(blocks, base[n], got):
            if len(b.channels) > 1:
                assert r == "mb"
            elif engine.block_parts(b).fused:
                assert r == "one"
            else:
                assert r == r0
    monkeypatch.setattr(engine, "SMALL_BATCH_RULE", True)
    monkeypatch.setattr(engine, "SMALL_BATCH_FASTER", ((("mb", 7, 2, True), 4), (("fused", 5, 1, True), 2)))
    for n in (1, 2, 4, 8):
        got = _routes(model, n)
        for b, r0, r in zip(blocks, base[1], got):
            kind = engine.small_batch_kind(b)
            if kind == ("mb", 7, 2, True) and n <= 4:
                assert r == "mb"
            elif kind == ("fused", 5, 1, True) and n <= 2:
                assert r == "one"
            else:
                assert r == r0, (kind, n)
    monkeypatch.setattr(engine, "EVAL_SMALL_BATCH", False)
    assert _routes(model, 1) == base[1]


class _Raises(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.seen = None

    def forward(self, x):
        self.seen = (engine.EVAL_SMALL_BATCH, engine.EVAL_MULTI_BRANCH)
        raise RuntimeError("model failed")


@pytest.mark.parametrize("small,fused", [(True, False), (False, False), (True, True)])
def test_eval_step_sets_the_switch_around_its_forward_only(small, fused):
    """EvalStep's eval body turns EVAL_SMALL_BATCH on for its forward and off afterwards, also
    when the forward raises; calibration does not touch it."""
    from yet_another_mobilenet_series_b200.trainer import EvalStep
    es = EvalStep.__new__(EvalStep)
    es.model = _Raises()
    es.small_batch, es.fused_multi_branch = small, fused
    with pytest.raises(RuntimeError, match="model failed"):
        es._eval_body(torch.zeros(1, 3, 8, 8), torch.zeros(1, dtype=torch.long))
    assert es.model.seen == (small, fused)
    assert engine.EVAL_SMALL_BATCH is False and engine.EVAL_MULTI_BRANCH is False
    with pytest.raises(RuntimeError, match="model failed"):
        es._calib_body(torch.zeros(1, 3, 8, 8), None)
    assert es.model.seen == (False, False)


def test_eval_step_default_is_off():
    import inspect
    from yet_another_mobilenet_series_b200.trainer import EvalStep
    assert inspect.signature(EvalStep).parameters["small_batch"].default is False


# ---- C ABI without a device ---------------------------------------------------------------------
def _mb_args():
    from yet_another_mobilenet_series_b200 import native as nat
    m = nat.BlockEvalMb()
    a = m.base
    a.N, a.H, a.W, a.Cin, a.Chid, a.Cout, a.kernel, a.stride, a.act = 1, 14, 14, 32, 256, 32, 7, 1, 3
    a.x = a.y = a.w_expand = a.w_project = a.pooled = 16
    a.w_dw = 16
    a.bn1.running_mean = a.bn1.running_var = a.bn2.running_mean = a.bn2.running_var = 16
    a.bn3.running_mean = a.bn3.running_var = 16
    m.ngroups, m.group_k[0], m.group_k[1], m.group_c0[1] = 2, 7, 3, 128
    return m


def test_abi_without_device(built_lib):
    from yet_another_mobilenet_series_b200 import native as nat
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = built_lib
    fns = (lib.yamb_block_eval_mb_cluster_fwd, lib.yamb_block_eval_mb_cluster_pool_fwd)
    for name in ("yamb_block_eval_mb_cluster_fwd", "yamb_block_eval_mb_cluster_pool_fwd"):
        assert name in nat.SYMBOLS and hasattr(lib, name)
    m = _mb_args()
    for fn in fns:
        assert fn(None, 2, None) == -1
        for cs in (2, 4, 8):
            assert fn(C.byref(m), cs, None) == -2          # YAMB_ENODEV
        for cs in (-1, 0, 1, 3, 16):
            assert fn(C.byref(m), cs, None) == -1
            assert b"cluster size" in lib.yamb_last_error()
        for bad in ({"ngroups": 0}, {"ngroups": 4}, {"group_k": (5, 3, 0)}, {"group_c0": (0, 12, 0)},
                    {"group_c0": (0, 256, 0)}, {"group_k": (7, 7, 0)}):
            b = nat.BlockEvalMb.from_buffer_copy(m)
            for field, v in bad.items():
                if isinstance(v, tuple):
                    for i, e in enumerate(v):
                        getattr(b, field)[i] = e
                else:
                    setattr(b, field, v)
            assert fn(C.byref(b), 2, None) == -1, bad
            assert b"block_eval_mb" in lib.yamb_last_error()
        b = nat.BlockEvalMb.from_buffer_copy(m)
        b.base.kernel = 3
        assert fn(C.byref(b), 4, None) == -1
        b = nat.BlockEvalMb.from_buffer_copy(m)
        b.base.w_expand = None
        assert fn(C.byref(b), 4, None) == -1


# ---- ptxas --------------------------------------------------------------------------------------
def test_instantiations_match_the_unsplit_launcher_and_spill_nothing(tmp_path):
    """block_eval_mb_cluster.cu names the geometries of block_eval_mb_launch, with CLUSTER; every
    (geometry, lean / generic activation, plain / gate / pool) kernel compiles without spills."""
    nvcc = os.environ.get("NVCC")
    if not (nvcc and os.path.exists(nvcc)):
        nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else \
            shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "yet_another_mobilenet_series_b200", "csrc", "block_eval_mb_cluster.cu")
    with open(src) as f:
        calls = re.findall(r"launch_eval<EvGeomMB<([\d,\s]+)>,\s*true,\s*true>", f.read())
    assert {tuple(int(v) for v in c.split(",")) for c in calls} == MB_GEOMS
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "mbc.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    kernels, cur = {}, None
    for line in (r.stdout + r.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1)
            kernels[cur] = []
            continue
        if cur:
            kernels[cur].append(line)
    pat = re.compile(r"EvGeomMBILi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)EEELb1ELb([01])"
                     r"ELi(\d)ELb1E")
    got = set()
    for name in kernels:
        m = pat.search(name)
        assert m, name
        v = tuple(int(g) for g in m.groups())
        got.add((v[:6], v[6], v[7]))
    assert got == {(g, lean, mode) for g in MB_GEOMS for lean in (0, 1) for mode in (0, 1, 2)}
    assert len(kernels) == 6 * 2 * 3
    for name, lines in kernels.items():
        props = " ".join(lines)
        assert "0 bytes spill stores, 0 bytes spill loads" in props, (name, props)
