"""CPU: the per-channel launchers of csrc/elementwise.cu (bn_apply, bn_stats, bn_reduce,
bn_bwd_apply, se_pool, se_bwd_reduce, se_bwd_apply) refuse malformed arguments with YAMB_EINVAL
before they look for a device, and the shape tables of tests/ew_cases.py cover the grid paths
they exist for.  Every call below is malformed in exactly one way; the pointers are fake, 16-byte
aligned device addresses that are never dereferenced."""
import ctypes as C

import pytest
import torch

import ew_cases as ec

_BASE = 1 << 20
_STEP = 0x100000


def _fill(s, ptrs, defaults=None, **kw):
    """Fake pointers for `ptrs`, then `defaults`, then the overrides `kw`."""
    for i, name in enumerate(ptrs):
        setattr(s, name, _BASE + i * _STEP)
    for k, v in dict(defaults or {}, **kw).items():
        setattr(s, k, v)
    return s


def _bn_bwd(nat):
    b = nat.BnBwd()
    return _fill(b, ("partials", "counter", "gamma", "mean", "invstd", "dgamma", "dbeta",
                     "ca", "cb", "cc"), count=64)


def _bn_fwd(nat):
    f = nat.BnFwd()
    return _fill(f, ("partials", "counter", "gamma", "beta", "scale", "shift", "mean", "invstd"),
                 count=64, eps=1e-3, momentum=0.1)


# (entry point, struct builder): the struct is well formed for M = 64 rows of C = 32 channels
def _apply(nat, **kw):
    return _fill(nat.BnApply(), ("h", "scale", "shift", "y"),
                 dict(M=64, C=32, ldh=32, ldr=32, ldy=32), **kw)


def _reduce(nat, **kw):
    r = _fill(nat.BnReduce(), ("dy", "h"), M=64, C=32, lddy=32, ldh=32)
    r.bn = C.pointer(_bn_bwd(nat))
    return _fill(r, (), **kw)


def _stats(nat, **kw):
    s = _fill(nat.BnStats(), ("h",), M=64, C=32, ldh=32)
    s.bn = C.pointer(_bn_fwd(nat))
    return _fill(s, (), **kw)


def _bwd_apply(nat, **kw):
    return _fill(nat.BnBwdApply(), ("dy", "h", "ca", "cb", "cc", "dh"),
                 dict(M=64, C=32, lddy=32, ldh=32, lddh=32), **kw)


def _pool(nat, **kw):
    return _fill(nat.SePool(), ("h", "scale", "shift", "pooled"), dict(N=2, HW=32, C=32, ldh=32),
                 **kw)


def _se_reduce(nat, **kw):
    return _fill(nat.SeBwdReduce(), ("dy", "h", "scale", "shift", "dgate"),
                 dict(N=2, HW=32, C=32, ldd=32, ldh=32), **kw)


def _se_apply(nat, **kw):
    a = _fill(nat.SeBwdApply(), ("dy", "h", "scale", "shift", "gate", "dpool", "dz"), M=64, C=32,
              ldd=32, ldh=32, ldz=32, rows_per_sample=32, ldg=32)
    a.bn = C.pointer(_bn_bwd(nat))
    return _fill(a, (), **kw)


_ODD = 8      # a base address 8 bytes past a 16-byte boundary

# entry point, builder, one defect per case: row pitch below C, a pitch that is not a multiple
# of 8 channels, a misaligned base for every bf16 operand read or written with 16-byte vectors
CASES = {
    "yamb_bn_apply_fwd": (_apply, [
        dict(C=12), dict(M=0), dict(ldh=24), dict(ldh=36), dict(ldy=24), dict(ldy=44),
        dict(h=_BASE + _ODD), dict(y=_BASE + 3 * _STEP + _ODD), dict(h=None), dict(y=None),
        dict(residual=_BASE + 5 * _STEP, ldr=24), dict(residual=_BASE + 5 * _STEP, ldr=36),
        dict(residual=_BASE + 5 * _STEP + _ODD),
        dict(residual2=_BASE + 6 * _STEP, ldr2=16), dict(residual2=_BASE + 6 * _STEP, ldr2=44),
        dict(residual2=_BASE + 6 * _STEP + _ODD, ldr2=32),
        dict(scale=_BASE + _STEP + 4), dict(shift=_BASE + 2 * _STEP + 8), dict(scale=None)]),
    "yamb_bn_stats_fwd": (_stats, [
        dict(C=12), dict(M=0), dict(ldh=24), dict(ldh=36), dict(h=_BASE + _ODD), dict(h=None),
        dict(bn=None)]),
    "yamb_bn_reduce_bwd": (_reduce, [
        dict(C=20), dict(lddy=24), dict(lddy=36), dict(ldh=16), dict(ldh=44),
        dict(dy=_BASE + _ODD), dict(h=_BASE + _STEP + _ODD), dict(dy=None), dict(bn=None),
        dict(z_scale=_BASE + 9 * _STEP, z_act=1)]),
    "yamb_bn_bwd_apply_bwd": (_bwd_apply, [
        dict(C=4), dict(lddy=24), dict(lddy=36), dict(ldh=16), dict(ldh=33), dict(lddh=24),
        dict(lddh=42), dict(dy=_BASE + _ODD), dict(h=_BASE + _STEP + _ODD),
        dict(dh=_BASE + 5 * _STEP + _ODD), dict(ca=None),
        dict(z_scale=_BASE + 9 * _STEP, z_act=2)]),
    "yamb_se_pool_fwd": (_pool, [
        dict(C=36), dict(HW=0), dict(ldh=24), dict(ldh=36), dict(h=_BASE + _ODD), dict(h=None),
        dict(N=65536)]),
    "yamb_se_bwd_reduce_bwd": (_se_reduce, [
        dict(C=36), dict(ldd=24), dict(ldd=36), dict(ldh=16), dict(ldh=44),
        dict(dy=_BASE + _ODD), dict(h=_BASE + _STEP + _ODD), dict(N=65536)]),
    "yamb_se_bwd_apply_bwd": (_se_apply, [
        dict(C=36), dict(rows_per_sample=0), dict(bn=None), dict(ldd=24), dict(ldd=36),
        dict(ldh=16), dict(ldh=44), dict(ldz=24), dict(ldz=52), dict(dy=_BASE + _ODD),
        dict(h=_BASE + _STEP + _ODD), dict(dz=_BASE + 6 * _STEP + _ODD), dict(dz=None),
        dict(gate=_BASE + 4 * _STEP + 4), dict(dpool=_BASE + 5 * _STEP + 8), dict(ldg=34)]),
}

_PARAMS = [(fn, i, bad) for fn, (_, bads) in CASES.items() for i, bad in enumerate(bads)]


def _refused(lib, rc):
    assert rc == -1, (rc, lib.yamb_last_error())
    assert lib.yamb_last_error() not in (b"", b"no CUDA device")


@pytest.mark.parametrize("fn,i,bad", _PARAMS, ids=["%s-%d" % (p[0][5:], p[1]) for p in _PARAMS])
def test_launcher_refuses(built_lib, fn, i, bad):
    from yet_another_mobilenet_series_b200 import native as nat
    make = CASES[fn][0]
    _refused(built_lib, getattr(built_lib, fn)(C.byref(make(nat, **bad)), None))


@pytest.mark.parametrize("fn", sorted(CASES))
def test_null_args(built_lib, fn):
    _refused(built_lib, getattr(built_lib, fn)(None, None))


@pytest.mark.parametrize("fn", sorted(CASES))
def test_well_formed_reaches_device_check(built_lib, fn):
    """The unmodified structs pass every argument check: without a device they get
    YAMB_ENODEV, so each refusal above is the check it names.  (With a device the fake pointers
    would be launched on, so this only runs where there is none.)"""
    if built_lib.yamb_max_ctas() > 0:
        pytest.skip("a CUDA device is visible")
    from yet_another_mobilenet_series_b200 import native as nat
    make = CASES[fn][0]
    extra = dict(residual=_BASE + 5 * _STEP, residual2=_BASE + 6 * _STEP, ldr2=32) \
        if fn == "yamb_bn_apply_fwd" else {}
    rc = getattr(built_lib, fn)(C.byref(make(nat, **extra)), None)
    assert rc == -2, (rc, built_lib.yamb_last_error())


def test_workspace_refuses_wider_batchnorm():
    """The statistics accumulator holds 2 * max_c doubles: a wider BatchNorm is refused before a
    kernel gets the buffer."""
    from yet_another_mobilenet_series_b200 import engine, native as nat
    ws = engine.Workspace.__new__(engine.Workspace)      # no device needed for the bound
    ws.max_c = 4096
    ws.partials = torch.zeros(4 * ws.max_c, dtype=torch.float32)
    ws.counter = torch.zeros(4, dtype=torch.int32)
    assert ws.partials.numel() * 4 == 2 * ws.max_c * 8
    assert ws.stats(4096) == (ws.partials.data_ptr(), ws.counter.data_ptr())
    with pytest.raises(nat.NativeError):
        ws.stats(4104)


# ------------------------------------------------------------------------------------------------
# the GPU case tables cover what they exist to cover
# ------------------------------------------------------------------------------------------------
def test_tables_cover_grid_paths():
    ec.check_tables(ec.H100_SMS)
