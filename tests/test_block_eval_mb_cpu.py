"""Multi-branch eval path (csrc/block_eval_mb.cu, engine.eval_forward_mb) without a GPU: the
packing algebra in fp64, the routing rule, the C ABI's argument checks and the ptxas report."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import torch_model as tm
from yet_another_mobilenet_series_b200 import engine
from yet_another_mobilenet_series_b200 import mobilenet_base as mb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BN = {"momentum": 0.01, "eps": 1e-3}
SWISH, RELU = mb.get_active_fn("nn.Swish"), mb.get_active_fn("nn.ReLU")
CONFIGS = ("atomnas_a", "atomnas_b", "atomnas_c", "atomnas_a+", "atomnas_b+", "atomnas_c+")


def load_cfgs():
    with open(os.path.join(ROOT, "tests", "golden", "model_cfgs_multi_branch.json")) as f:
        return json.load(f)


def build(name):
    from yet_another_mobilenet_series_b200 import searched_network  # noqa: F401
    import importlib
    cfg = load_cfgs()[name]
    lib = importlib.import_module(cfg["flags"]["model"].replace(
        "models.", "yet_another_mobilenet_series_b200."))
    torch.manual_seed(0)
    return lib.Model(**cfg["model_kwparams"], input_size=cfg["flags"]["image_size"])


def multi_branch_blocks(model):
    return [m for m in model.modules()
            if isinstance(m, (mb.InvertedResidualChannels, mb.InvertedResidualChannelsFused))
            and len(m.channels) > 1]


def randomise(block, gen):
    """Random weights and running statistics (fp64 module)."""
    with torch.no_grad():
        for p in block.parameters():
            p.copy_(torch.randn(p.shape, generator=gen, dtype=p.dtype) * 0.3)
        for m in block.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.copy_(torch.randn(m.num_features, generator=gen, dtype=m.running_mean.dtype) * 0.2)
                m.running_var.copy_(torch.rand(m.num_features, generator=gen, dtype=m.running_var.dtype) + 0.5)
    return block.eval()


def packed_forward(block, x):
    """The packed single-branch block the kernels run, restated in fp64: gather every tensor
    through engine.mb_layout's map, zero-embed the taps in K_MAX x K_MAX, run each 64-channel slice
    with the stencil of the group of its first channel over the centred window."""
    parts = engine.block_parts(block)
    lay = engine.mb_layout(block.kernel_sizes, block.channels)
    K, Chid, dt = lay.kmax, lay.Chid, x.dtype
    offs = [sum(block.channels[:i]) for i in range(len(block.channels))]
    W1 = torch.zeros(Chid, block.input_dim, dtype=dt)
    W3 = torch.zeros(block.output_dim, Chid, dtype=dt)
    taps = torch.zeros(Chid, K, K, dtype=dt)
    bn1 = torch.zeros(4, Chid, dtype=dt)
    bn2 = torch.zeros(4, Chid, dtype=dt)
    bn1[3] = bn2[3] = 1.0
    se = parts.se
    if se is not None:
        R = se.se_reduce.weight.shape[0]
        Wr, We, be = torch.zeros(R, Chid, dtype=dt), torch.zeros(Chid, R, dtype=dt), torch.zeros(Chid, dtype=dt)
    code = torch.tensor(lay.map)
    for b in range(len(block.channels)):
        js = torch.nonzero((code >= 0) & ((code >> 16) == b)).flatten()
        c = code[js] & 0xFFFF
        k = block.kernel_sizes[b]
        if parts.fused:
            src, e1, w3, b1 = offs[b] + c, parts.expand_convs[0], parts.project_convs[0], parts.bn1s[0]
        else:
            src, e1, w3, b1 = c, parts.expand_convs[b], parts.project_convs[b], parts.bn1s[b]
        W1[js] = e1.weight[src, :, 0, 0]
        W3[:, js] = w3.weight[:, src, 0, 0]
        o = (K - k) // 2
        conv_d, b2 = parts.dws[b]
        taps[js, o:o + k, o:o + k] = conv_d.weight[c, 0]
        for dst, bn, i in ((bn1, b1, src), (bn2, b2, c)):
            dst[:, js] = torch.stack([bn.weight[i], bn.bias[i], bn.running_mean[i], bn.running_var[i]])
        if se is not None:
            Wr[:, js] = se.se_reduce.weight[:, offs[b] + c, 0, 0]
            We[js] = se.se_expand.weight[offs[b] + c, :, 0, 0]
            be[js] = se.se_expand.bias[offs[b] + c]
    eps = parts.dws[0][1].eps
    act = block.active_fn()
    fold = lambda bn, h: (h - bn[2][None, :, None, None]) / torch.sqrt(bn[3] + eps)[None, :, None, None] * \
        bn[0][None, :, None, None] + bn[1][None, :, None, None]
    a1 = act(fold(bn1, torch.einsum("nchw,dc->ndhw", x, W1)))
    s = block.stride
    outs = []
    for c0 in range(0, Chid, 64):
        kc = [k for k, g0 in lay.groups if g0 <= c0][-1]
        o = (K - kc) // 2
        w = taps[c0:c0 + 64, o:o + kc, o:o + kc].unsqueeze(1)
        outs.append(F.conv2d(a1[:, c0:c0 + 64], w, stride=s, padding=(kc - 1) // 2, groups=w.shape[0]))
    a2 = act(fold(bn2, torch.cat(outs, 1)))
    if se is not None:
        pooled = a2.mean((2, 3))
        se_act = se.active_fn if isinstance(se.active_fn, torch.nn.Module) else se.active_fn()
        v = se_act(pooled @ Wr.t() + se.se_reduce.bias)
        a2 = a2 * torch.sigmoid(v @ We.t() + be)[:, :, None, None]
    y = parts.bn3(torch.einsum("nchw,dc->ndhw", a2, W3))
    return y + x if block.use_res_connect else y


def reference_forward(block, x):
    fwd = tm._fused_forward if hasattr(block, "expand_conv") else tm._unfused_forward
    return types.MethodType(fwd, block)(x)


def _check_algebra(block, H, gen):
    block = randomise(block.double(), gen)
    x = torch.randn(2, block.input_dim, H, H, generator=gen, dtype=torch.float64)
    with torch.no_grad():
        want, got = reference_forward(block, x), packed_forward(block, x)
    assert got.shape == want.shape
    assert (got - want).abs().max().item() <= 1e-12 * max(1.0, want.abs().max().item())


@pytest.mark.parametrize("name", CONFIGS)
def test_packing_algebra_every_multi_branch_block(name):
    """Every multi-branch block of the config: the packed block in fp64 equals the module's own
    eval forward (SE included for the '+' configs)."""
    model = build(name)
    blocks = multi_branch_blocks(model)
    assert blocks
    gen = torch.Generator().manual_seed(1)
    for block in blocks:
        _check_algebra(block, 9 if block.stride == 1 else 10, gen)


@pytest.mark.parametrize("fused", [False, True])
def test_packing_algebra_slices_straddle_groups(fused):
    """Odd branch widths whose padded groups start inside 64-channel slices (7 | 5 boundary at 72,
    5 | 3 boundary at 136), the supernet's three branches of expand ratio 6, stride 1 and 2."""
    gen = torch.Generator().manual_seed(2)
    cls = mb.InvertedResidualChannelsFused if fused else mb.InvertedResidualChannels
    kw = {"se_ratio": 0.25} if fused else {}
    for inp, oup, s, ch, ks in ((24, 24, 1, [37, 61, 70], [3, 5, 7]),
                                (24, 32, 2, [71, 13], [7, 3]),
                                (16, 24, 2, [96, 96, 96], [3, 5, 7]),
                                (32, 32, 1, [192, 192], [5, 3])):
        block = cls(inp, oup, s, ch, ks, True, active_fn=SWISH, batch_norm_kwargs=BN, **kw)
        _check_algebra(block, 9, gen)


def test_layout():
    lay = engine.mb_layout([3, 5, 7], [13, 20, 9])
    assert lay.kmax == 7 and lay.Chid == 16 + 24 + 16
    assert lay.groups == [(7, 0), (5, 16), (3, 40)]
    assert lay.map[:9] == [(2 << 16) | c for c in range(9)] and lay.map[9:16] == [-1] * 7
    assert lay.map[16:36] == [(1 << 16) | c for c in range(20)] and lay.map[36:40] == [-1] * 4
    assert engine.mb_layout([3, 3], [8, 16]).groups == [(3, 0)]


# ---- routing ------------------------------------------------------------------------------------
# The blocks of every config that take the multi-branch path with EVAL_MULTI_BRANCH on, in module
# order ((K_MAX, stride, fused class) kinds MB_SHAPE_RULE keeps, BASELINE.md §5).
def _routed(model):
    x = torch.zeros(2, 8, 14, 14)
    out = []
    for i, block in enumerate(multi_branch_blocks(model)):
        if engine.eval_mb_supported(block, x):
            out.append(i)
    return out


def test_flag_off_by_default():
    assert engine.EVAL_MULTI_BRANCH is False and engine.MB_SHAPE_RULE is True
    block = mb.InvertedResidualChannelsFused(40, 40, 1, [40, 24, 32], [3, 5, 7], True,
                                             active_fn=SWISH, batch_norm_kwargs=BN).eval()
    with torch.no_grad():
        assert not engine.eval_mb_supported(block, torch.zeros(2, 40, 14, 14))


def test_predicate(monkeypatch):
    monkeypatch.setattr(engine, "EVAL_MULTI_BRANCH", True)
    monkeypatch.setattr(engine, "MB_SHAPE_RULE", False)
    x = torch.zeros(2, 40, 14, 14)
    f = lambda *a, **kw: mb.InvertedResidualChannelsFused(
        *a, active_fn=kw.pop("act", SWISH), batch_norm_kwargs=BN, **kw).eval()
    u = lambda *a: mb.InvertedResidualChannels(*a, active_fn=RELU, batch_norm_kwargs=BN).eval()
    ok = f(40, 40, 1, [40, 23, 28], [3, 5, 7], True, se_ratio=0.25)
    assert not engine.eval_mb_supported(ok, x)      # gradient mode
    with torch.no_grad():
        assert engine.eval_mb_supported(ok, x)
        assert engine.eval_mb_supported(f(40, 48, 2, [120, 120], [3, 5], True), x)
        assert engine.eval_mb_supported(u(40, 40, 1, [40, 24], [7, 3], True), x)
        assert not engine.eval_mb_supported(f(40, 40, 1, [40], [3], True), x)          # one branch
        assert not engine.eval_mb_supported(f(40, 40, 1, [40, 40], [3, 3], True), x)   # K_MAX 3
        assert not engine.eval_mb_supported(f(40, 40, 1, [40, 40], [3, 5], False), x)  # no expansion
        assert not engine.eval_mb_supported(f(264, 264, 1, [64, 64], [3, 5], True), x)
        assert not engine.eval_mb_supported(f(40, 44, 1, [64, 64], [3, 5], True), x)
        assert not engine.eval_mb_supported(f(40, 40, 1, [64, 64], [3, 5], True, nl_c=0.25, nl_s=1), x)
        trained = f(40, 40, 1, [64, 64], [3, 5], True)
        trained.depth_ops[1][1][1].train()
        assert not engine.eval_mb_supported(trained, x)
    monkeypatch.setattr(engine, "EVAL_MULTI_BRANCH", False)
    with torch.no_grad():
        assert not engine.eval_mb_supported(ok, x)


ROUTED = {name: [] for name in CONFIGS}


@pytest.mark.parametrize("name", CONFIGS)
def test_shape_rule_per_config(monkeypatch, name):
    monkeypatch.setattr(engine, "EVAL_MULTI_BRANCH", True)
    model = build(name).eval()
    with torch.no_grad():
        got = _routed(model)
        kinds = sorted({engine.mb_kind(b) for b in multi_branch_blocks(model)})
    assert got == [i for i, b in enumerate(multi_branch_blocks(model))
                   if engine.mb_kind(b) in engine.MB_FASTER], (name, kinds)
    assert got == ROUTED[name], (name, got)


# ---- C ABI without a device ---------------------------------------------------------------------
def test_abi_without_device(built_lib):
    from yet_another_mobilenet_series_b200 import native as nat
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = built_lib
    for name in ("yamb_block_eval_mb_pack", "yamb_block_eval_mb_fwd", "yamb_block_eval_mb_pool_fwd"):
        assert name in nat.SYMBOLS and hasattr(lib, name)
    m = nat.BlockEvalMb()
    a = m.base
    a.N, a.H, a.W, a.Cin, a.Chid, a.Cout, a.kernel, a.stride, a.act = 2, 14, 14, 32, 128, 32, 7, 1, 3
    a.x = a.y = a.w_expand = a.w_project = 16
    a.w_dw = 16
    a.bn1.running_mean = a.bn1.running_var = a.bn2.running_mean = a.bn2.running_var = 16
    a.bn3.running_mean = a.bn3.running_var = 16
    m.ngroups, m.group_k[0], m.group_k[1], m.group_c0[1] = 2, 7, 3, 64
    for fn in (lib.yamb_block_eval_mb_fwd, lib.yamb_block_eval_mb_pool_fwd):
        assert fn(None, None) == -1
        assert fn(C.byref(m), None) == -2        # YAMB_ENODEV
    pk = nat.BlockEvalMbPack()
    assert lib.yamb_block_eval_mb_pack(None, None) == -1
    pk.Cin, pk.Cout, pk.nbranch, pk.Chid, pk.kmax = 32, 32, 4, 8, 3
    assert lib.yamb_block_eval_mb_pack(C.byref(pk), None) == -1
    assert b"branches" in lib.yamb_last_error()


# ---- ptxas --------------------------------------------------------------------------------------
# block_eval_kernel<EvGeomMB<K, S, TOH, TOW, TI, CPT>, EXPAND, LEAN, MODE, CLUSTER> the launcher
# names (block_eval_mb_launch)
MB_GEOMS = {(5, 2, 6, 7, 1, 2), (5, 1, 7, 7, 1, 4), (5, 1, 7, 16, 1, 4), (5, 1, 7, 7, 2, 4),
            (7, 2, 4, 7, 1, 2), (7, 1, 7, 7, 1, 2)}


def test_instantiations_match_the_launcher_and_spill_nothing(tmp_path):
    nvcc = os.environ.get("NVCC")
    if not (nvcc and os.path.exists(nvcc)):
        nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else \
            shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "yet_another_mobilenet_series_b200", "csrc", "block_eval_mb.cu")
    with open(src) as f:
        calls = re.findall(r"launch_eval<EvGeomMB<([\d,\s]+)>,\s*true,\s*false>", f.read())
    assert {tuple(int(v) for v in c.split(",")) for c in calls} == MB_GEOMS
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "mb.o")],
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
                     r"ELi(\d)ELb0E")
    got = set()
    for name in kernels:
        if "block_eval_kernel" not in name:
            assert "block_eval_mb_pack_kernel" in name, name
            continue
        m = pat.search(name)
        assert m, name
        v = tuple(int(g) for g in m.groups())
        got.add((v[:6], v[6], v[7]))
    assert got == {(g, lean, mode) for g in MB_GEOMS for lean in (0, 1) for mode in (0, 1, 2)}
    assert len(kernels) == 6 * 2 * 3 + 1
    for name, lines in kernels.items():
        props = " ".join(lines)
        assert "0 bytes spill stores, 0 bytes spill loads" in props, (name, props)
