"""yamb_expand_bwd (csrc/expand_bwd.cu) without a device: the plan query, the refusals, which
blocks the engine sends to it, and the ptxas report of every instantiation."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "yet_another_mobilenet_series_b200", "csrc", "expand_bwd.cu")


def _nat():
    from yet_another_mobilenet_series_b200 import native as nat
    return nat


def _args(M=3211264, Cin=16, Chid=96):
    a = _nat().ExpandBwd()
    a.M, a.Cin, a.Chid = M, Cin, Chid
    return a


def _plan(lib, a, sms=132):
    info = _nat().ExpandBwdPlanInfo()
    rc = lib.yamb_expand_bwd_plan(C.byref(a), sms, C.byref(info))
    return rc, info


def test_struct_sizes(built_lib):
    nat = _nat()
    assert built_lib.yamb_struct_size(29) == C.sizeof(nat.ExpandBwd)
    assert built_lib.yamb_struct_size(30) == C.sizeof(nat.ExpandBwdPlanInfo)


@pytest.mark.parametrize("M,Cin,Chid,block_n,panels", [
    (3211264, 16, 96, 16, 2), (802816, 24, 144, 32, 3), (200704, 32, 192, 32, 3),
    (128, 8, 64, 16, 1), (1000, 32, 128, 32, 2)])
def test_plan(built_lib, M, Cin, Chid, block_n, panels):
    nat = _nat()
    rc, info = _plan(built_lib, _args(M, Cin, Chid))
    assert rc == 0
    assert (info.block_n, info.panels) == (block_n, panels)
    # the slabs are the split-K wgrad GEMM's (the plan of the launch the kernel replaces): dW1 is
    # summed per slab in the same order, so it is bitwise the two-GEMM path's
    g = nat.Gemm()
    g.M, g.N, g.K = Chid, Cin, M
    g.a_mn_major = g.b_mn_major = 1
    g.epi, g.a_xform = 2, 2
    g.a_scale = g.a_shift = g.a_scale2 = g.A2 = 4096   # the plan checks presence, not values
    wi = nat.GemmPlanInfo()
    assert built_lib.yamb_gemm_plan(C.byref(g), 132, C.byref(wi)) == 0
    assert (info.slabs, info.slab_rows) == (wi.ksplit, wi.kb_per_split * 64)
    assert (info.slabs - 1) * info.slab_rows < M <= info.slabs * info.slab_rows
    assert info.grid == min(info.slabs, 132)
    # the stage ring fills the 227 KB that the x ring, W1 and the barriers leave
    assert 4 <= info.num_stages <= 6
    assert info.smem_bytes <= 232448


@pytest.mark.parametrize("edit", [dict(M=0), dict(M=-5), dict(Cin=0), dict(Cin=12), dict(Cin=40),
                                  dict(Chid=48), dict(Chid=100), dict(Chid=200)])
def test_refused_shapes(built_lib, edit):
    a = _args()
    for k, v in edit.items():
        setattr(a, k, v)
    rc, _ = _plan(built_lib, a)
    assert rc == _nat().EINVAL
    # the launch refuses the same arguments before touching a device
    assert built_lib.yamb_expand_bwd(C.byref(a), None) == _nat().EINVAL


def test_refused_pointers(built_lib):
    nat = _nat()
    a = _args()
    a.dz1 = a.h1 = a.ca = a.cb = a.cc = a.W1 = a.x = a.dx = a.dW1 = 4096
    a.dz1 = None
    assert built_lib.yamb_expand_bwd(C.byref(a), None) == nat.EINVAL
    a.dz1 = 4096 + 8                       # not 16-byte aligned
    assert built_lib.yamb_expand_bwd(C.byref(a), None) == nat.EINVAL
    a.dz1, a.residual = 4096, 4096 + 2
    assert built_lib.yamb_expand_bwd(C.byref(a), None) == nat.EINVAL
    assert b"expand_bwd" in built_lib.yamb_last_error()


def _expand_blocks(config, batch):
    """(M_in, Cin, Chid) of every expanding block of a bench configuration at `batch`."""
    import bench
    model = bench.build_model(config=config)
    H = 224 // 2                           # after the stride-2 stem
    out = []
    for m in model.modules():
        if hasattr(m, "use_res_connect") and hasattr(m, "channels"):
            if m.expand:
                out.append((batch * H * H, m.input_dim, sum(m.channels)))
            H = (H - 1) // m.stride + 1
    assert H == 7
    return out


def test_fused_blocks_of_the_bench_configurations(built_lib):
    import sys
    sys.path.insert(0, ROOT)
    import bench
    from yet_another_mobilenet_series_b200 import engine
    taken = {}
    for config, (_, batch) in bench.CONFIGS.items():
        blocks = _expand_blocks(config, batch)
        taken[config] = [b for b in blocks if engine.expand_bwd_fused(*b)]
        for b in taken[config]:
            assert b[0] >= engine.EXPAND_BWD_MIN_M and 8 <= b[1] <= 32 and 64 <= b[2] <= 192
    # MobileNetV2-1.0 at N = 256: blocks 2-7 (112^2, 56^2, 28^2 input maps)
    assert taken["mobilenet_v2"] == [(256 * 112 * 112, 16, 96), (256 * 56 * 56, 24, 144),
                                     (256 * 56 * 56, 24, 144), (256 * 28 * 28, 32, 192),
                                     (256 * 28 * 28, 32, 192), (256 * 28 * 28, 32, 192)]


def test_launch_args_cases_stay_on_two_gemms(built_lib):
    from yet_another_mobilenet_series_b200 import engine
    # tests/test_launch_args_gpu.py: N = 2 at 8 x 8, Cin 16, hidden 48; and a 128-pixel block that
    # the kernel would cover
    assert not engine.expand_bwd_fused(2 * 8 * 8, 16, 48)
    assert not engine.expand_bwd_fused(2 * 8 * 8, 16, 96)


def _nvcc():
    env = os.environ.get("NVCC")
    if env and os.path.exists(env):
        return env
    if os.path.exists("/usr/local/cuda/bin/nvcc"):
        return "/usr/local/cuda/bin/nvcc"
    return shutil.which("nvcc")


def test_ptxas_no_spills_no_serialised_wgmma(tmp_path):
    nvcc = _nvcc()
    if not nvcc:
        pytest.skip("nvcc not found")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xptxas", "-v", "-c", SRC, "-o", str(tmp_path / "expand_bwd.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    report = r.stdout + r.stderr
    kernels = {}
    cur = None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1) if "expand_bwd_kernel" in m.group(1) else None
            if cur:
                kernels[cur] = []
            continue
        if cur:
            kernels[cur].append(line)
    # wgmma width 16 / 32 x one, two or three panels
    assert len(kernels) == 6, sorted(kernels)
    for name, lines in kernels.items():
        text = "\n".join(lines)
        assert "0 bytes spill stores" in text and "0 bytes spill loads" in text, (name, text)
    assert "C7510" not in report and "C7520" not in report, report[-4000:]
