"""CPU: the GPU tables of tests/tail_cases.py reach every path of the stem convolution, softmax
cross entropy and column-sum kernels, and their launchers refuse malformed arguments with
YAMB_EINVAL before they look for a device.  Every refused call below is malformed in exactly one
way; the pointers are fake, 16-byte aligned device addresses that are never dereferenced."""
import ctypes as C

import pytest

import tail_cases as tc

SMS = tc.H100_SMS


# ---- the GPU tables cover the kernels' paths -------------------------------------------------------
def test_stem_plan():
    p = tc.stem_plan(66, 230, 230)
    assert (p.Ho, p.Wo, p.tiles_h, p.tiles_w, p.num_tiles, p.aligned) == (115, 115, 8, 4, 2112, True)
    p = tc.stem_plan(66, 225, 225)
    assert (p.Ho, p.Wo, p.tiles_h, p.tiles_w, p.num_tiles, p.aligned) == (113, 113, 8, 4, 2112, False)
    p = tc.stem_plan(64, 224, 224)
    assert (p.Ho, p.tiles_h, p.num_tiles) == (112, 7, 64 * 28) and not tc.stem_cut_edges(p)
    assert tc.stem_plan(1, 1, 1)[:5] == (1, 1, 1, 1, 1)
    assert tc.stem_wgrad_slots(396, 32) == 396 * 8 and tc.stem_wgrad_slots(264, 64) == 264 * 4


def test_stem_forward_table():
    paths = {(c.Cout, tc.stem_plan(c.N, c.H, c.W).aligned) for c in tc.STEM_CASES}
    assert paths >= {(co, al) for co in tc.STEM_FWD_COUT for al in (True, False)}
    fwd_walks = {(c.Cout, tc.stem_plan(c.N, c.H, c.W).aligned) for c in tc.STEM_WALK_CASES}
    assert fwd_walks >= {(co, al) for co in (8, 64) for al in (True, False)}
    # tiny images: every H and W in 1..3
    tiny = [c for c in tc.STEM_CASES if c.H <= 3 and c.W <= 3]
    assert {c.H for c in tiny} == {1, 2, 3} and {c.W for c in tiny} == {1, 2, 3}
    for c in tc.STEM_CASES + tc.STEM_WALK_CASES:
        assert c.Cout in tc.STEM_FWD_COUT
        assert (c.N + 1) * c.H * c.W * 3 <= 12 * 2 ** 20, c         # moderate test data
    assert set(tc.STEM_EVAL_COUT) >= {24, 56}
    assert {tc.stem_plan(*s).aligned for s in tc.STEM_EVAL_SHAPES} == {True, False}


def test_stem_wgrad_walks():
    walks = set()
    for c in tc.STEM_WALK_CASES:
        p = tc.stem_plan(c.N, c.H, c.W)
        assert tc.stem_is_walk(p, SMS), c
        assert tc.stem_cut_edges(p), ("walk without cut last tiles", c)
        walks.add((c.Cout, p.aligned))
    assert walks == {(co, al) for co in tc.STEM_WGRAD_COUT for al in (True, False)}
    # the direct cases stay direct: the walks are what makes a CTA cover several tiles
    assert not any(tc.stem_is_walk(tc.stem_plan(c.N, c.H, c.W), SMS) for c in tc.STEM_CASES)


def test_loss_table():
    cs = tc.CE_CASES
    Cs = {c.C for c in cs}
    assert Cs >= {1, 2, 4, 5, 6, tc.CE_MAX_C}
    assert any(c.C % 32 for c in cs) and any(c.C % 32 == 0 for c in cs)
    assert any(c.C % 2 for c in cs), "odd C in the forward"
    assert any(c.N % 8 for c in cs)
    assert all(c.C <= tc.CE_MAX_C and c.ld >= c.C and c.ldg >= c.C and c.ldd >= c.C for c in cs)
    assert any(c.ld > c.C for c in cs) and any(c.ldg > c.C for c in cs)
    assert {c.eps for c in cs} == {0.0, 0.1}
    bwd = [c for c in cs if tc.ce_has_bwd(c)]
    assert any(c.ldd > c.C for c in bwd)
    # the backward's grid-stride row loop and several column pairs per thread, with dbias
    assert any(c.N > tc.ce_bwd_grid(c.N, SMS) for c in bwd)
    assert any(tc.pairs_per_thread(c.C) > 1 for c in bwd)
    assert any(c.N > 2 * SMS and tc.pairs_per_thread(c.C) > 1 for c in bwd)
    assert tc.ce_bwd_grid(600, SMS) == 264 and tc.ce_fwd_grid(13) == 2
    assert tc.pairs_per_thread(1000) == 2 and tc.pairs_per_thread(4096) == 8


def test_colsum_table():
    cs = tc.COLSUM_CASES
    Ms = {c.M for c in cs}
    assert any(m < 32 for m in Ms) and 32 in Ms and any(m > 32 for m in Ms)
    assert any(tc.colsum_grid(c.M, c.C)[0] > 1 for c in cs)       # C / 2 > 256
    assert any(c.ld > c.C for c in cs) and any(c.ld == c.C for c in cs)
    for c in cs:
        assert c.C % 2 == 0 and c.ld % 2 == 0 and c.ld >= c.C
    assert tc.colsum_grid(4097, 1280) == (3, 32) and tc.colsum_grid(1, 2) == (1, 1)


# ---- launcher validation -----------------------------------------------------------------------------
_BASE = 1 << 20
_STEP = 0x100000
_ODD = 8          # 8 bytes past a 16-byte boundary


def _stem(nat, **kw):
    a = nat.StemConv()
    a.N, a.H, a.W, a.Cout = 2, 37, 37, 32
    a.x, a.w, a.y, a.dh, a.dw = (_BASE + i * _STEP for i in range(5))
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _stem_eval(nat, conv=None, **kw):
    e = nat.StemConvEval()
    e.conv = _stem(nat, **(conv or {}))
    e.scale, e.shift, e.act = _BASE + 5 * _STEP, _BASE + 6 * _STEP, 1
    for k, v in kw.items():
        setattr(e, k, v)
    return e


def _ce(nat, **kw):
    a = nat.SoftmaxCe()
    a.N, a.C, a.ld, a.ldg, a.smoothing = 16, 1000, 1000, 1000, 0.1
    a.logits, a.target, a.loss, a.correct1, a.correct5, a.G = (_BASE + i * _STEP for i in range(6))
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _ce_grad(nat, **kw):
    a = nat.SoftmaxCeGrad()
    a.N, a.C, a.ldg, a.ldd = 16, 1000, 1000, 1000
    a.G, a.dloss, a.dlogits, a.dbias = (_BASE + i * _STEP for i in range(4))
    for k, v in kw.items():
        setattr(a, k, v)
    return a


_SHAPES = [dict(Cout=0), dict(Cout=12), dict(Cout=72), dict(N=0), dict(H=0), dict(W=-1),
           dict(x=None)]
STEM_FWD = _SHAPES + [dict(y=None), dict(y=_BASE + 2 * _STEP + _ODD), dict(w=None)]
STEM_WGRAD = _SHAPES + [dict(Cout=24), dict(Cout=40), dict(Cout=48), dict(Cout=56),
                        dict(dh=None), dict(dh=_BASE + 3 * _STEP + _ODD), dict(dw=None)]
STEM_EVAL = [dict(conv=b) for b in STEM_FWD] + [dict(act=5), dict(act=-1), dict(scale=None),
                                                dict(shift=None)]
CE_FWD = [dict(C=4097), dict(C=0), dict(N=0), dict(ld=999), dict(ldg=999), dict(logits=None),
          dict(target=None), dict(loss=None)]
CE_BWD = [dict(C=999, ldg=1000, ldd=1000), dict(ldg=1001), dict(ldd=1003), dict(ldg=998),
          dict(ldd=998), dict(N=0), dict(G=None), dict(dloss=None), dict(dlogits=None),
          dict(G=_BASE + 2), dict(dlogits=_BASE + 2 * _STEP + 2)]
# (M, C, ld, X): odd C, odd ld, ld < C, no rows, misaligned X
COLSUM = [(64, 999, 1000, _BASE), (64, 1000, 1001, _BASE), (64, 1000, 998, _BASE),
          (0, 1000, 1000, _BASE), (64, 1000, 1000, _BASE + 2), (64, 1000, 1000, None)]


def _refused(lib, rc):
    assert rc == -1, (rc, lib.yamb_last_error())
    assert lib.yamb_last_error() not in (b"", b"no CUDA device")


def _ids(prefix, cases):
    return ["%s-%d" % (prefix, i) for i in range(len(cases))]


@pytest.mark.parametrize("bad", STEM_FWD, ids=_ids("fwd", STEM_FWD))
def test_stem_fwd_refuses(built_lib, bad):
    from yet_another_mobilenet_series_b200 import native as nat
    _refused(built_lib, built_lib.yamb_stem_conv_fwd(C.byref(_stem(nat, **bad)), None))


@pytest.mark.parametrize("bad", STEM_WGRAD, ids=_ids("wgrad", STEM_WGRAD))
def test_stem_wgrad_refuses(built_lib, bad):
    from yet_another_mobilenet_series_b200 import native as nat
    _refused(built_lib, built_lib.yamb_stem_conv_wgrad(C.byref(_stem(nat, **bad)), None))


@pytest.mark.parametrize("bad", STEM_EVAL, ids=_ids("eval", STEM_EVAL))
def test_stem_eval_refuses(built_lib, bad):
    from yet_another_mobilenet_series_b200 import native as nat
    _refused(built_lib, built_lib.yamb_stem_conv_eval_fwd(C.byref(_stem_eval(nat, **bad)), None))


@pytest.mark.parametrize("bad", CE_FWD, ids=_ids("fwd", CE_FWD))
def test_ce_fwd_refuses(built_lib, bad):
    from yet_another_mobilenet_series_b200 import native as nat
    _refused(built_lib, built_lib.yamb_softmax_ce_fwd(C.byref(_ce(nat, **bad)), None))


@pytest.mark.parametrize("bad", CE_BWD, ids=_ids("bwd", CE_BWD))
def test_ce_bwd_refuses(built_lib, bad):
    from yet_another_mobilenet_series_b200 import native as nat
    _refused(built_lib, built_lib.yamb_softmax_ce_bwd(C.byref(_ce_grad(nat, **bad)), None))


@pytest.mark.parametrize("M,Cc,ld,X", COLSUM, ids=_ids("colsum", COLSUM))
def test_colsum_refuses(built_lib, M, Cc, ld, X):
    _refused(built_lib, built_lib.yamb_colsum_bf16(X, M, Cc, ld, _BASE + 4 * _STEP, None))


def test_null_args(built_lib):
    for fn in ("yamb_stem_conv_fwd", "yamb_stem_conv_wgrad", "yamb_stem_conv_eval_fwd",
               "yamb_softmax_ce_fwd", "yamb_softmax_ce_bwd"):
        _refused(built_lib, getattr(built_lib, fn)(None, None))


def test_well_formed_reaches_device_check(built_lib):
    """The unmodified arguments pass every check: without a device they get YAMB_ENODEV, so each
    refusal above is the check it names.  (With a device the fake pointers would be launched on,
    so this only runs where there is none.)"""
    if built_lib.yamb_max_ctas() > 0:
        pytest.skip("a CUDA device is visible")
    from yet_another_mobilenet_series_b200 import native as nat
    lib = built_lib
    calls = [lib.yamb_stem_conv_fwd(C.byref(_stem(nat)), None),
             lib.yamb_stem_conv_wgrad(C.byref(_stem(nat)), None),
             lib.yamb_stem_conv_fwd(C.byref(_stem(nat, Cout=24)), None),
             lib.yamb_stem_conv_eval_fwd(C.byref(_stem_eval(nat, conv=dict(Cout=56))), None),
             lib.yamb_softmax_ce_fwd(C.byref(_ce(nat, C=4096, ld=4096, ldg=4096)), None),
             lib.yamb_softmax_ce_fwd(C.byref(_ce(nat, C=5, ld=5, G=None, ldg=0)), None),
             lib.yamb_softmax_ce_bwd(C.byref(_ce_grad(nat)), None),
             lib.yamb_colsum_bf16(_BASE, 64, 1000, 1000, _BASE + 4 * _STEP, None)]
    for i, rc in enumerate(calls):
        assert rc == -2, (i, rc, lib.yamb_last_error())
