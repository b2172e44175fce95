"""CPU: the pointwise GEMM case table (tests/gemm_cases.py) reaches every compiled gemm_tc_kernel
instantiation and every axis of the launch plan, read from the library's own plan query
(yamb_gemm_plan, 132 SMs, no device), and the plan refuses malformed arguments with the launch's
codes and messages.  The instantiation list is parsed out of csrc/gemm_tc.cu, so adding a pick_tc /
launch_tc without a case fails here; YAMB_GEMM_SOURCE points the parser at another copy of the
source."""
import ctypes as C
import os

import pytest

import gemm_cases as gc

SOURCE = os.environ.get("YAMB_GEMM_SOURCE") or gc.GEMM_SOURCE


@pytest.fixture(scope="module")
def plans(built_lib):
    from yet_another_mobilenet_series_b200 import native as nat
    out = {}
    for c in gc.CASES:
        rc, info = gc.plan(built_lib, nat, c)
        assert rc == 0, (c.name, built_lib.yamb_last_error())
        out[c.name] = info
    return out


def test_instantiations_parse():
    inst = gc.compiled_instantiations(SOURCE)
    assert len(inst) == len(set(inst)) == 11, inst


def test_table_reaches_every_instantiation(plans):
    reached = {gc.inst_of(p) for p in plans.values()}
    missing = sorted(set(gc.compiled_instantiations(SOURCE)) - reached)
    assert missing == [], "instantiations without a case: %s" % missing
    assert reached <= set(gc.compiled_instantiations(gc.GEMM_SOURCE))


def _cases(plans, pred):
    return [c.name for c in gc.CASES if pred(c, plans[c.name])]


def test_table_reaches_every_plan_axis(plans):
    need = {
        # transformed operands: register and TMA loaders, modes 1 and 2, with and without a gate
        "A mode 1 reg": lambda c, p: c.a_xform == 1 and not p.a_tma and not c.gate,
        "A mode 1 tma": lambda c, p: c.a_xform == 1 and p.a_tma and not c.gate,
        "A mode 1 reg gate": lambda c, p: c.a_xform == 1 and not p.a_tma and c.gate,
        "A mode 1 tma gate": lambda c, p: c.a_xform == 1 and p.a_tma and c.gate,
        "A mode 2 reg": lambda c, p: c.a_xform == 2 and not p.a_tma,
        "A mode 2 tma": lambda c, p: c.a_xform == 2 and p.a_tma,
        "B mode 1 reg": lambda c, p: c.b_xform == 1 and not p.b_tma and not c.gate,
        "B mode 1 tma": lambda c, p: c.b_xform == 1 and p.b_tma and not c.gate,
        "B mode 1 reg gate": lambda c, p: c.b_xform == 1 and not p.b_tma and c.gate,
        "B mode 1 tma gate": lambda c, p: c.b_xform == 1 and p.b_tma and c.gate,
        "B mode 2 reg": lambda c, p: c.b_xform == 2 and not p.b_tma,
        "B mode 2 tma": lambda c, p: c.b_xform == 2 and p.b_tma,
        "wg2x 0 (transform)": lambda c, p: (c.a_xform or c.b_xform) and not p.wg2x,
        "wg2x 1": lambda c, p: p.wg2x == 1,
        "wg2x 1 epi 0": lambda c, p: p.wg2x == 1 and c.epi == 0,
        "lgroup 1": lambda c, p: p.lgroup == 1,
        "lgroup 2": lambda c, p: p.lgroup == 2,
        "lgroup 4": lambda c, p: p.lgroup == 4,
        "out_bufs 1": lambda c, p: p.out_bufs == 1 and c.epi != 2,
        "out_bufs 2": lambda c, p: p.out_bufs == 2 and c.epi != 2,
        "out_bufs 1, epi 1, N ~ 960, two-source A":
            lambda c, p: p.out_bufs == 1 and c.epi == 1 and c.N >= 900 and c.a_xform == 2,
        "ksplit 1": lambda c, p: p.ksplit == 1,
        "ksplit > 1, uneven last slab":
            lambda c, p: p.ksplit > 1 and p.num_k_blocks % p.kb_per_split != 0,
        "simple_work": lambda c, p: p.simple_work == 1,
        "not simple_work": lambda c, p: p.simple_work == 0,
        ">= 2 tiles per CTA, odd tile count":
            lambda c, p: gc.tiles_per_cta(p) >= 2 and p.num_work % 2 == 1 and c.epi != 2,
        "reg_stats epi 0": lambda c, p: p.reg_stats == 1 and c.epi == 0,
        "reg_stats epi 1": lambda c, p: p.reg_stats == 1 and c.epi == 1,
        "reg_stats over a walk": lambda c, p: p.reg_stats == 1 and gc.tiles_per_cta(p) >= 4,
        "shared statistics": lambda c, p: (c.stats or c.epi == 1) and not p.reg_stats,
        "last m-block <= 64 rows": lambda c, p: c.M % 128 != 0 and c.M % 128 <= 64 and c.epi != 2,
        "MN-major A <= 64 rows": lambda c, p: c.a_mn and c.M <= 64,
        "gate rows_per_sample 1": lambda c, p: c.gate == 1,
        "gate rows_per_sample 49": lambda c, p: c.gate == 49,
        "gate rows_per_sample 196": lambda c, p: c.gate == 196,
        "gate rows_per_sample 200": lambda c, p: c.gate == 200,
        "strided operands and a channel slice": lambda c, p: c.pad > 0 and c.c0 > 0,
        "sliced epi 1": lambda c, p: c.epi == 1 and c.c0 > 0,
        "sliced epi 2": lambda c, p: c.epi == 2 and c.c0 > 0,
        "momentum None": lambda c, p: c.stats and c.mom is None,
        "momentum 0.1": lambda c, p: c.stats and c.mom == 0.1,
        "momentum 0.01": lambda c, p: c.stats and c.mom == 0.01,
        "NULL gamma / beta": lambda c, p: (c.stats or c.epi == 1) and not c.affine,
        "NULL running statistics": lambda c, p: c.stats and not c.running,
        "use_batch_stats 0": lambda c, p: c.epi == 1 and c.use_batch_stats == 0,
        "NULL dgamma / dbeta": lambda c, p: c.epi == 1 and not c.grads,
        "long chain": lambda c, p: c.shifted and c.M >= 500000 and p.reg_stats,
    }
    for k in (8, 16, 24, 40, 56):
        need["K %% 64 = %d" % k] = lambda c, p, k=k: c.K % 64 == k
    missing = [axis for axis, pred in need.items() if not _cases(plans, pred)]
    assert missing == [], "plan axes no case reaches: %s" % missing


def test_max_ctas_changes_ksplit(built_lib, plans):
    from yet_another_mobilenet_series_b200 import native as nat
    found = False
    for c in gc.CASES:
        if c.epi == 2 and c.max_ctas:
            _, free = gc.plan(built_lib, nat, c, max_ctas=0)
            found |= plans[c.name].ksplit > 1 and plans[c.name].ksplit != free.ksplit
    assert found, "no split-K case whose max_ctas changes ksplit"


def test_plan_matches_the_documented_rules(plans):
    """A few facts of the plan the kernels rely on (an MN-major B always has block_n 64; the
    statistics are register-resident exactly when there is one n-block)."""
    for c in gc.CASES:
        p = plans[c.name]
        assert p.grid == min(p.num_work, c.max_ctas or gc.PLAN_SMS), c.name
        assert p.num_work == p.m_blocks * p.n_blocks * p.ksplit, c.name
        assert (p.ksplit - 1) * p.kb_per_split < p.num_k_blocks <= p.ksplit * p.kb_per_split, c.name
        if c.b_mn:
            assert p.block_n == 64, c.name
        assert 2 <= p.num_stages <= 8 and p.lgroup in (1, 2, 4) and p.out_bufs in (1, 2), c.name
        assert p.smem_bytes <= 232448 - 2048, c.name
        assert p.reg_stats == int((c.stats or c.epi == 1) and p.n_blocks == 1), c.name


def test_case_data_fits(plans):
    for c in gc.CASES:
        assert gc.est_bytes(c) <= gc.MAX_BYTES, (c.name, gc.est_bytes(c))
        assert c.pad % 8 == 0 and c.c0 % 8 == 0, c.name


def test_plan_without_device_uses_given_sms(built_lib):
    from yet_another_mobilenet_series_b200 import native as nat
    c = gc.BY_NAME["plain_big"]
    _, p132 = gc.plan(built_lib, nat, c, sms=132)
    _, p7 = gc.plan(built_lib, nat, c, sms=7)
    assert p132.grid == 132 and p7.grid == 7


# ------------------------------------------------------------------------------------------------
# refusals: each call is malformed in one way and refused with YAMB_EINVAL and the launch's message
# ------------------------------------------------------------------------------------------------
_BASE = gc.BY_NAME["stats"]
_REFUSALS = [
    ("N % 8", dict(N=100), "multiples of 8"),
    ("K % 8, K-major A", dict(K=20), "multiples of 8"),
    ("M % 8, MN-major A", dict(M=44, N=16, K=640, a_mn=1, b_mn=1, epi=2, stats=False),
     "multiples of 8"),
    ("K % 8, K-major B", dict(K=44, b_mn=1), "multiples of 8"),
    ("bad epilogue", dict(epi=3, stats=False), "bad epilogue"),
    ("epi 0, MN-major A", dict(a_mn=1, M=64), "layout not supported"),
    ("epi 1, K-major B", dict(epi=1, stats=False), "layout not supported"),
    ("epi 1, MN-major A", dict(epi=1, a_mn=1, b_mn=1, M=64, stats=False), "layout not supported"),
    ("epi 2, K-major A", dict(epi=2, b_mn=1, stats=False), "layout not supported"),
    ("epi 2, K-major B", dict(epi=2, a_mn=1, M=64, stats=False), "layout not supported"),
]


@pytest.mark.parametrize("what,kw,msg", _REFUSALS, ids=[r[0] for r in _REFUSALS])
def test_plan_refusals_shape_layout(built_lib, what, kw, msg):
    from dataclasses import replace
    from yet_another_mobilenet_series_b200 import native as nat
    c = replace(_BASE, **kw)
    rc, _ = gc.plan(built_lib, nat, c)
    assert rc == -1 and msg.encode() in built_lib.yamb_last_error(), (what, rc,
                                                                       built_lib.yamb_last_error())


def _refused(lib, nat, c, drop=(), msg=b"", **set_fields):
    from yet_another_mobilenet_series_b200 import native as nat  # noqa: F811
    ptrs = gc.fake_ptrs(c)
    for k in drop:
        ptrs.pop(k)
    g = gc.gemm_struct(nat, c, ptrs)
    for k, v in set_fields.items():
        setattr(g, k, v)
    rc, _ = gc.plan(lib, nat, c, g=g)
    assert rc == -1 and msg in lib.yamb_last_error(), (rc, lib.yamb_last_error())


def test_plan_refusals_arguments(built_lib):
    from dataclasses import replace
    from yet_another_mobilenet_series_b200 import native as nat
    x1 = gc.BY_NAME["xform1"]
    _refused(built_lib, nat, x1, drop=("a_scale",), msg=b"transform without coefficients")
    _refused(built_lib, nat, x1, drop=("a_shift",), msg=b"transform without coefficients")
    wx = gc.BY_NAME["wgrad_xform"]
    _refused(built_lib, nat, wx, drop=("b_shift",), msg=b"transform without coefficients")
    x2 = gc.BY_NAME["xform2"]
    _refused(built_lib, nat, x2, drop=("A2",), msg=b"two-source transform without second")
    _refused(built_lib, nat, x2, drop=("a_scale2",), msg=b"two-source transform without second")
    b2 = gc.BY_NAME["wgrad_b2_reg_n24"]
    _refused(built_lib, nat, b2, drop=("B2",), msg=b"two-source transform without second")
    gate = gc.BY_NAME["proj_gate_reg_k40"]
    _refused(built_lib, nat, gate, msg=b"gate without gate_rows_per_sample", gate_rows_per_sample=0)
    wg = gc.BY_NAME["wgrad_gate_reg_n40"]
    _refused(built_lib, nat, wg, msg=b"gate without gate_rows_per_sample", gate_rows_per_sample=0)
    # b_gate on a K-major B (forward with a transformed B)
    kb = replace(gc.BY_NAME["plain_small"], b_xform=1, act=1)
    _refused(built_lib, nat, kb, msg=b"b_gate needs an MN-major B", b_gate=gc._FAKE,
             gate_rows_per_sample=64)
    dz = gc.BY_NAME["dz"]
    for k in ("H", "h_scale", "h_shift"):
        _refused(built_lib, nat, dz, drop=(k,), msg=b"dz epilogue needs H")
    g = gc.gemm_struct(nat, dz, gc.fake_ptrs(dz))
    info = nat.GemmPlanInfo()
    assert built_lib.yamb_gemm_plan(C.byref(g), 132, C.byref(info)) == -1   # no bn_bwd
    assert b"dz epilogue needs" in built_lib.yamb_last_error()
    assert built_lib.yamb_gemm_plan(None, 132, C.byref(info)) == -1
    assert built_lib.yamb_gemm_plan(C.byref(g), 132, None) == -1
