"""CPU: the non-local block with `nl_norm: nn.InstanceNorm`.

The InstanceNorm oracle (tests/nl_instancenorm_oracle.py) against the live reference's records
(tests/golden/blocks_nl_in.pt), the eval dispatch rule, the C ABI of the two new entry points and
the ptxas report of csrc/instance_norm.cu."""
import os
import re
import shutil
import subprocess

import pytest
import torch

import nl_instancenorm_oracle as no
from oracle import ir_block as ob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, b):
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.fixture(scope="module")
def golden():
    return no.load_golden()


@pytest.mark.parametrize("name", [c[0] for c in no.CASES])
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_oracle_matches_reference(golden, name, mode):
    rec = golden[name]
    blk = no.build_block(rec)
    assert isinstance(blk.nl_op.bn, torch.nn.InstanceNorm2d)
    cfg, P = no.extract(blk)
    tr = mode == "train"
    y, S = no.forward(rec["x"], cfg, P, training=tr)
    dx, G = no.backward(rec[mode]["dy"], cfg, P, S, training=tr)
    gold = rec[mode]
    assert _rel(y, gold["y"]) < 2e-6
    assert _rel(dx, gold["dx"]) < 5e-6
    got = no.named_grads(cfg, G)
    assert set(got) == set(dict(blk.named_parameters()))
    for k, g in got.items():
        assert _rel(g.reshape(gold["grads"][k].shape), gold["grads"][k]) < 2e-5, k
    after = gold["state_after"]
    if tr:
        assert _rel(S["bn4_rm_after"], after["nl_op.bn.running_mean"]) < 1e-5
        assert _rel(S["bn4_rv_after"], after["nl_op.bn.running_var"]) < 1e-5
        # BN3 of the same block: the ordinary BatchNorm bookkeeping
        rm, rv, _ = ob.bn_running_update(P["bn3_rm"], P["bn3_rv"], S["bn3_mean"], S["bn3_var"],
                                         S["count_out"], cfg.momentum, 0)
        assert _rel(rm, after["project_conv.1.running_mean"]) < 1e-5
        assert _rel(rv, after["project_conv.1.running_var"]) < 1e-5
    else:
        assert torch.equal(after["nl_op.bn.running_mean"], rec["state"]["nl_op.bn.running_mean"])
    # InstanceNorm never counts batches
    assert int(after["nl_op.bn.num_batches_tracked"]) == \
        int(rec["state"]["nl_op.bn.num_batches_tracked"])


def test_quant_mode_is_close_to_fp32(golden):
    rec = golden["in_autonl_7x7"]
    cfg, P = no.extract(no.build_block(rec))
    y, S = no.forward(rec["x"], cfg, P, training=True)
    yq, Sq = no.forward(rec["x"], cfg, P, training=True, quant=True)
    dx, _ = no.backward(rec["train"]["dy"], cfg, P, S, training=True)
    dxq, _ = no.backward(rec["train"]["dy"], cfg, P, Sq, training=True, quant=True)
    assert _rel(yq, y) < 2e-2 and _rel(dxq, dx) < 5e-2


def _in_block(training):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    blk = mb.InvertedResidualChannelsFused(24, 24, 1, [72], [3], True, mb.get_active_fn("nn.Swish"),
                                           {"momentum": 0.01, "eps": 1e-3}, nl_c=0.25, nl_s=1)
    blk.nl_op.bn = mb.get_nl_norm_fn("nn.InstanceNorm")(24, momentum=0.01, eps=1e-3)
    return blk.train(training)


def test_fused_class_eval_dispatch():
    from yet_another_mobilenet_series_b200 import engine
    x = torch.zeros(2, 24, 14, 14)
    blk = _in_block(False)
    with torch.no_grad():
        assert engine.fused_class_eval_supported(blk, x)
    assert not engine.fused_class_eval_supported(blk, x)      # a gradient is wanted
    with torch.no_grad():
        assert not engine.fused_class_eval_supported(_in_block(True), x)
        blk.nl_op.bn.train()                                  # InstanceNorm alone in train mode
        assert not engine.fused_class_eval_supported(blk, x)
        blk.nl_op.bn.eval()
        blk.nl_op.bn = torch.nn.GroupNorm(4, 24).eval()
        assert not engine.fused_class_eval_supported(blk, x)
        blk.nl_op.bn = torch.nn.InstanceNorm2d(24, affine=True).eval()     # untracked
        assert not engine.fused_class_eval_supported(blk, x)


def test_unsupported_norms_raise():
    from yet_another_mobilenet_series_b200 import engine, native
    for norm in (torch.nn.GroupNorm(4, 24), torch.nn.InstanceNorm2d(24, affine=True),
                 torch.nn.InstanceNorm2d(24, track_running_stats=True)):
        assert not engine._nl_norm_supported(norm)
    assert engine._nl_norm_supported(_in_block(True).nl_op.bn)
    assert engine._nl_norm_supported(torch.nn.BatchNorm2d(24))
    assert issubclass(native.NativeError, RuntimeError)


def test_struct_sizes_and_load_without_driver(built_lib):
    from yet_another_mobilenet_series_b200 import native
    assert built_lib.yamb_struct_size(22) == __import__("ctypes").sizeof(native.InFwd)
    assert built_lib.yamb_struct_size(23) == __import__("ctypes").sizeof(native.InBwd)
    assert hasattr(built_lib, "yamb_instance_norm_fwd")
    assert hasattr(built_lib, "yamb_instance_norm_bwd")
    if not torch.cuda.is_available():
        s = native.InFwd()
        s.N, s.HW, s.C, s.ldh, s.ldy = 2, 49, 24, 24, 24
        s.h = s.y = s.mean = s.invstd = 16
        assert built_lib.yamb_instance_norm_fwd(s, None) == -2          # YAMB_ENODEV
        s.HW = 1
        assert built_lib.yamb_instance_norm_fwd(s, None) == -1          # YAMB_EINVAL: H*W = 1


def _nvcc():
    env = os.environ.get("NVCC")
    if env and os.path.exists(env):
        return env
    if os.path.exists("/usr/local/cuda/bin/nvcc"):
        return "/usr/local/cuda/bin/nvcc"
    return shutil.which("nvcc")


def test_ptxas_no_spills(tmp_path):
    nvcc = _nvcc()
    if not nvcc:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "yet_another_mobilenet_series_b200", "csrc", "instance_norm.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "in.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    report = r.stdout + r.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)'", report)
    assert len(kernels) == 2 and all("in_fwd_kernel" in k or "in_bwd_kernel" in k
                                     for k in kernels), kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", report)
    assert len(spills) == 2 and all(a == "0" and b == "0" for a, b in spills), report
