"""CPU: the depthwise GPU test table reaches every compiled kernel instantiation at a shape where
each CTA walks at least two tiles, and the launchers reject malformed arguments before they look
for a device.  The dispatch itself is restated in tests/dw_cases.py; the instantiation list is
parsed out of the CUDA sources, so adding a YAMB_FWD_CASE / YAMB_DW_BWD without a test case fails
here."""
import ctypes as C
import os

import pytest

import dw_cases as dc

# the instantiation list can be pointed at other copies of the sources (a scratch edit that adds
# one) to check that this test notices
_SRC_ENV = os.environ.get("YAMB_DW_SOURCES")
SOURCES = _SRC_ENV.split(os.pathsep) if _SRC_ENV else dc.DW_SOURCES


def _plans(c):
    return (dc.fwd_plan(c.N, c.H, c.W, c.C, c.k, c.s), dc.bwd_plan(c.N, c.H, c.W, c.C, c.k, c.s))


def test_instantiations_parse():
    fwd, bwd = dc.compiled_instantiations(SOURCES)
    assert len(fwd) == len(set(fwd)) and len(bwd) == len(set(bwd))
    assert len(fwd) == 40 and len(bwd) == 24, (len(fwd), len(bwd))
    # every parsed tuple is one the host dispatch can select
    for k, s, ct, tw in fwd:
        assert k in (3, 5, 7) and s in (1, 2) and ct in (8, 16, 32, 64) and tw in (1, 2)
        assert not (k == 7 and tw == 2)
    for k, s, ct in bwd:
        assert k in (3, 5, 7) and s in (1, 2) and ct in (8, 16, 32, 64)


def test_walk_table_reaches_every_instantiation():
    fwd, bwd = dc.compiled_instantiations(SOURCES)
    walk_f, walk_b = set(), set()
    for c in dc.WALK_CASES:
        f, b = _plans(c)
        Ho, Wo = dc.out_size(c.H, c.k, c.s), dc.out_size(c.W, c.k, c.s)
        if dc.is_walk(f):
            assert dc.partial_tiles(f, Ho, Wo), ("forward walk without partial last tiles", c)
            walk_f.add(f.inst)
        if dc.is_walk(b):
            assert dc.partial_tiles(b, c.H, c.W), ("backward walk without partial last tiles", c)
            walk_b.add(b.inst)
    assert sorted(set(fwd) - walk_f) == [], "forward kernels without a walk case"
    assert sorted(set(bwd) - walk_b) == [], "backward kernels without a walk case"
    # nothing in the table selects a kernel that is not compiled
    assert walk_f <= set(fwd) and walk_b <= set(bwd)


def test_walk_table_edges():
    cases = dc.WALK_CASES
    assert any(_plans(c)[0].chunks > 1 and _plans(c)[1].chunks > 1 for c in cases)
    assert any(c.c0 > 0 and c.c0 + c.C < c.ldc for c in cases)
    assert any(c.s == 2 and c.H % 2 == 1 and c.W % 2 == 1 for c in cases)
    for c in cases:
        assert c.C % 8 == 0 and c.c0 % 8 == 0 and c.ldc % 8 == 0 and c.c0 + c.C <= c.ldc
        assert c.N * c.H * c.W * c.ldc <= 12 * 2 ** 20, c     # moderate test data
    # every activation code with the producer's BatchNorm prologue; identity inputs too
    assert {c.act for c in cases if c.pro} == {0, 1, 2, 3, 4}
    assert any(not c.pro for c in cases)
    assert {c.mom for c in cases} == {0.1, -1.0}


def test_pick_ct_and_tw():
    # rows: Ho in the forward, H in the backward (stride 2 can split them)
    assert dc.fwd_plan(1, 40, 40, 8, 3, 2).ct == 16 and dc.bwd_plan(1, 40, 40, 8, 3, 2).ct == 8
    assert [dc.pick_ct(c, 56) for c in (8, 16, 24, 32, 40, 64, 96, 144, 160, 192)] == \
        [8, 16, 32, 32, 64, 64, 32, 32, 32, 64]
    assert dc.pick_ct(8, 27) == 16 and dc.pick_ct(8, 13) == 32 and dc.pick_ct(16, 13) == 32
    assert dc.fwd_plan(1, 16, 16, 64, 3, 2).tw == 1        # Wo = 8
    assert dc.fwd_plan(1, 18, 18, 64, 3, 2).tw == 2        # Wo = 9
    assert dc.fwd_plan(1, 56, 56, 64, 7, 1).tw == 1        # k = 7
    p = dc.fwd_plan(3, 57, 59, 96, 5, 1)                  # ct 32: 16 x 16 output tiles
    assert (p.tile_h, p.tile_w, p.tiles_h, p.tiles_w, p.chunks) == (16, 16, 4, 4, 3)
    assert p.num_tiles == 3 * 3 * 4 * 4
    b = dc.bwd_plan(3, 57, 59, 96, 5, 1)
    assert (b.tile_h, b.tile_w, b.tiles_h, b.tiles_w, b.num_tiles) == (16, 8, 4, 8, 3 * 3 * 4 * 8)


# ------------------------------------------------------------------------------------------------
# launcher validation: every call below is malformed in exactly one way and must be refused with
# YAMB_EINVAL before any device is touched (the pointers are never dereferenced)
# ------------------------------------------------------------------------------------------------
_BASE = 1 << 20     # fake, 16-byte aligned device addresses


def _fwd(nat, **kw):
    d = nat.DwFwd()
    d.N, d.H, d.W, d.C, d.ldc, d.k, d.stride = 2, 16, 16, 32, 32, 3, 1
    d.x, d.y, d.w = _BASE, _BASE + 0x100000, _BASE + 0x200000
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _bwd(nat, **kw):
    e = nat.DwBwd()
    e.N, e.H, e.W, e.C, e.ldc, e.k, e.stride = 2, 16, 16, 32, 32, 3, 1
    ptrs = ("dz", "h", "ca", "cb", "cc", "w", "dw", "x", "dx", "residual")
    for i, name in enumerate(ptrs):
        setattr(e, name, _BASE + i * 0x100000)
    for k, v in kw.items():
        setattr(e, k, v)
    return e


_SHAPE_ERRORS = [dict(C=12), dict(C=32, ldc=24), dict(C=16, ldc=36), dict(k=1), dict(k=4),
                 dict(stride=3), dict(C=4104, ldc=4104), dict(N=0), dict(H=0)]


def _refused(lib, rc):
    assert rc == -1, (rc, lib.yamb_last_error())
    assert lib.yamb_last_error() not in (b"", b"no CUDA device")


@pytest.mark.parametrize("bad", _SHAPE_ERRORS + [dict(x=None), dict(y=None), dict(w=None),
                                                 dict(x=_BASE + 8), dict(y=_BASE + 0x100008)])
def test_fwd_validation(built_lib, bad):
    from yet_another_mobilenet_series_b200 import native as nat
    _refused(built_lib, built_lib.yamb_depthwise_fwd(C.byref(_fwd(nat, **bad)), None))


@pytest.mark.parametrize("bad", _SHAPE_ERRORS + [
    dict(dz=None), dict(h=None), dict(x=None), dict(dx=None), dict(dw=None), dict(w=None),
    dict(ca=None), dict(cb=None), dict(cc=None),
    dict(dz=_BASE + 8), dict(h=_BASE + 0x100008), dict(x=_BASE + 0x700008),
    dict(dx=_BASE + 0x800002), dict(residual=_BASE + 0x900002)])
def test_bwd_validation(built_lib, bad):
    from yet_another_mobilenet_series_b200 import native as nat
    _refused(built_lib, built_lib.yamb_depthwise_bwd(C.byref(_bwd(nat, **bad)), None))


def test_null_args(built_lib):
    _refused(built_lib, built_lib.yamb_depthwise_fwd(None, None))
    _refused(built_lib, built_lib.yamb_depthwise_bwd(None, None))
