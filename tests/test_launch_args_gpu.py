"""GPU: the host-side arguments of every kernel launch the engine makes, pinned.

Small seeded blocks and ConvBNReLU layers run one training forward + backward (and the fused-class
block one no_grad eval forward) with `engine.launch` / `engine.try_launch` wrapped by a recorder
that calls the real function.  Per call it keeps the entry point, the tag and cost numbers, the
stream it went to (the current one or the weight-gradient side stream) and every field of the
argument struct: the value of each non-pointer field, only NULL or not for each pointer, and the
BatchNorm sub-structs reached through `bn`, `bn_fwd` and `bn_bwd` the same way.  The records must
equal tests/golden/launch_args.json entry by entry: the numerical tests only see what these
arguments do, this test sees the arguments themselves.

Rewrite the golden (only when a launch is meant to change):
    python tests/test_launch_args_gpu.py [OUT.json]
"""
import ctypes as C
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "launch_args.json")
BN = {"momentum": 0.01, "eps": 1e-3}

pytestmark = pytest.mark.gpu


def _fields(st):
    out = {}
    for name, typ in st._fields_:
        v = getattr(st, name)
        if typ is C.c_void_p:
            out[name] = None if v is None else "ptr"
        elif issubclass(typ, C._Pointer):
            out[name] = _fields(v.contents) if v else None
        elif issubclass(typ, C.Structure):
            out[name] = _fields(v)
        else:
            out[name] = v
    return out


def _recorder(engine, real, log):
    def rec(fn, st, tag="", nbytes=0, flops=0):
        cur = torch.cuda.current_stream()
        side = any(s["stream"] == cur for s in engine._side.values())
        log.append({"fn": fn.__name__, "tag": tag, "nbytes": nbytes, "flops": flops,
                    "stream": "side" if side else "current", "args": _fields(st)})
        return real(fn, st, tag, nbytes, flops)
    return rec


# ---- cases: (module factory, input shape, train) -------------------------------------------------
def _ir(*args):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    return mb.InvertedResidualChannels(*args, active_fn=mb.get_active_fn("nn.ReLU"),
                                       batch_norm_kwargs=BN)


def _fused(nl_norm):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    blk = mb.InvertedResidualChannelsFused(16, 16, 1, [48], [3], True, mb.get_active_fn("nn.Swish"),
                                           BN, se_ratio=0.25, nl_c=0.25, nl_s=1)
    blk.nl_op.bn = mb.get_nl_norm_fn(nl_norm)(16, **BN)
    return blk


def _fused_branches():
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    return mb.InvertedResidualChannelsFused(16, 24, 2, [16, 24], [3, 5], True,
                                            mb.get_active_fn("nn.Swish"), BN, se_ratio=0.25)


def _conv_bn_relu(*args, **kw):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    return mb.ConvBNReLU(*args, active_fn=mb.get_active_fn("nn.ReLU6"), batch_norm_kwargs=BN, **kw)


CASES = {
    "ir_expand_s1": (lambda: _ir(16, 16, 1, [48], [3], True), (2, 16, 8, 8), True),
    "ir_expand_s2": (lambda: _ir(16, 24, 2, [48], [5], True), (2, 16, 8, 8), True),
    "ir_no_expand_s1": (lambda: _ir(16, 16, 1, [16], [3], False), (2, 16, 8, 8), True),
    "ir_no_expand_s2": (lambda: _ir(16, 24, 2, [16], [3], False), (2, 16, 8, 8), True),
    "ir_branches": (lambda: _ir(16, 16, 1, [16, 24], [3, 5], True), (2, 16, 8, 8), True),
    "ir_padded": (lambda: _ir(16, 16, 1, [15, 23, 13], [3, 5, 7], True), (2, 16, 8, 8), True),
    "fused_se_nl_bn": (lambda: _fused("nn.BatchNorm"), (2, 16, 8, 8), True),
    "fused_se_nl_in": (lambda: _fused("nn.InstanceNorm"), (2, 16, 8, 8), True),
    "fused_branches_se": (_fused_branches, (2, 16, 8, 8), True),
    "stem": (lambda: _conv_bn_relu(3, 16, 3, 2), (2, 3, 16, 16), True),
    "head": (lambda: _conv_bn_relu(32, 64, 1), (2, 32, 4, 4), True),
    "fused_se_nl_bn_eval": (lambda: _fused("nn.BatchNorm"), (2, 16, 8, 8), False),
    "fused_se_nl_in_eval": (lambda: _fused("nn.InstanceNorm"), (2, 16, 8, 8), False),
}


def record(name):
    """Every launch one run of CASES[name] makes, in order."""
    from yet_another_mobilenet_series_b200 import engine
    make, shape, train = CASES[name]
    torch.manual_seed(1995)
    mod = make().cuda().train(train)
    x = torch.randn(shape).cuda()
    log = []
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(engine, "SIDE_WGRAD", True)
        mp.setattr(engine, "DEFER_JOIN", False)
        mp.setattr(engine, "PROFILE", None)
        mp.setattr(engine, "EVAL_FUSED", True)
        mp.setattr(engine, "launch", _recorder(engine, engine.launch, log))
        mp.setattr(engine, "try_launch", _recorder(engine, engine.try_launch, log))
        if train:
            y = mod(x.requires_grad_(True))
            y.backward(torch.randn(y.shape).to(y.device, y.dtype))
        else:
            with torch.no_grad():
                mod(x)
        torch.cuda.synchronize()
    return log


def _first_difference(got, want, path="args"):
    if isinstance(want, dict) and isinstance(got, dict):
        for k in sorted(set(got) | set(want)):
            if got.get(k) != want.get(k):
                return _first_difference(got.get(k), want.get(k), path + "." + k)
    return "%s: %r, golden %r" % (path, got, want)


@pytest.mark.parametrize("name", list(CASES))
def test_launch_args(built_lib, name):
    with open(GOLDEN) as f:
        want = json.load(f)[name]
    got = json.loads(json.dumps(record(name)))   # the golden's number types
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, "launch %d (%s): %s" % (i, w["tag"], _first_difference(g, w, "launch"))
    assert len(got) == len(want), [r["tag"] for r in got]


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    out = sys.argv[1] if len(sys.argv) > 1 else GOLDEN
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with open(out, "w") as f:
        json.dump({name: record(name) for name in CASES}, f, indent=1)
        f.write("\n")
    print("wrote", out)
