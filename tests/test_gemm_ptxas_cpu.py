"""ptxas report of the pointwise GEMM (csrc/gemm_tc.cu): every gemm_tc_kernel instantiation keeps
its wgmma sequence pipelined (no C7510 / C7520 serialisation warning) and spills nothing.

Compiles for sm_90a without a GPU; skipped where no nvcc is installed."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "yet_another_mobilenet_series_b200", "csrc", "gemm_tc.cu")


def _nvcc():
    env = os.environ.get("NVCC")
    if env and os.path.exists(env):
        return env
    if os.path.exists("/usr/local/cuda/bin/nvcc"):
        return "/usr/local/cuda/bin/nvcc"
    return shutil.which("nvcc")


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    nvcc = _nvcc()
    if not nvcc:
        pytest.skip("nvcc not found")
    out = str(tmp_path_factory.mktemp("ptxas") / "gemm_tc.o")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xptxas", "-v", "-c", SRC, "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout + r.stderr


def _kernels(report):
    """{mangled gemm_tc_kernel name: its 'Function properties' lines}"""
    found = {}
    cur = None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1) if "gemm_tc_kernel" in m.group(1) else None
            if cur:
                found[cur] = []
            continue
        if cur:
            found[cur].append(line)
    return found


def test_every_instantiation_compiled(ptxas_report):
    kernels = _kernels(ptxas_report)
    # forward (block_n 16 / 32 / 64) and dgrad (+ residual) x transform, dz epilogue, wgrad x transform
    assert len(kernels) == 11, sorted(kernels)


def test_no_wgmma_serialisation(ptxas_report):
    bad = [l for l in ptxas_report.splitlines()
           if ("C7510" in l or "C7520" in l) and "gemm_tc_kernel" in l]
    assert not bad, "\n".join(bad)


def test_no_spills(ptxas_report):
    kernels = _kernels(ptxas_report)
    assert kernels
    for name, lines in kernels.items():
        props = " ".join(lines)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", props)
        assert m, (name, props)
        assert m.group(1) == "0" and m.group(2) == "0", (name, props)
