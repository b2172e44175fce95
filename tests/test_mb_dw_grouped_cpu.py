"""CPU: the grouped depthwise launches of multi-branch training blocks (TrainStep(grouped_branches=
True)): the grouping plan of every multi-branch block of AtomNAS-A/B/C(+) and of the [3, 5, 7]
supernet, the ABI struct mirror, the host validation of yamb_depthwise_fwd_grouped / _bwd_grouped
without a device, and that the switch is set only inside the step."""
import ctypes as C
import inspect
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_cfg(name):
    """Model and config of an AtomNAS configuration (tests/golden/model_cfgs_multi_branch.json)."""
    import importlib
    import json
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    from yet_another_mobilenet_series_b200 import searched_network  # noqa: F401
    with open(os.path.join(ROOT, "tests", "golden", "model_cfgs_multi_branch.json")) as f:
        cfg = json.load(f)[name]
    lib = importlib.import_module(cfg["flags"]["model"].replace(
        "models.", "yet_another_mobilenet_series_b200."))
    torch.manual_seed(0)
    model = lib.Model(**cfg["model_kwparams"], input_size=cfg["flags"]["image_size"])
    model.apply(mb.init_weights_mnas)
    return model, cfg


def test_switch_off_by_default_and_set_only_inside_the_step():
    from yet_another_mobilenet_series_b200 import engine, trainer
    assert engine.TRAIN_MB_DW_GROUPED is False
    assert inspect.signature(trainer.TrainStep).parameters["grouped_branches"].default is False
    src = inspect.getsource(trainer.TrainStep._fwd_bwd)
    on = src.index("engine.TRAIN_MB_DW_GROUPED = self.grouped_branches")
    fin = src.index("finally:")
    assert on < src.index("self._passes(") < fin
    assert "engine.TRAIN_MB_DW_GROUPED = False" in src[fin:]
    whole = inspect.getsource(trainer)
    assert whole.count("engine.TRAIN_MB_DW_GROUPED =") == 2
    for fn in ("state_dict", "load_state_dict", "save_status"):
        if hasattr(trainer.TrainStep, fn):
            assert "grouped_branches" not in inspect.getsource(getattr(trainer.TrainStep, fn))


def test_struct_sizes(built_lib):
    from yet_another_mobilenet_series_b200 import native as nat
    assert built_lib.yamb_struct_size(41) == C.sizeof(nat.DwFwdGrouped)
    assert built_lib.yamb_struct_size(42) == C.sizeof(nat.DwBwdGrouped)
    for name in ("yamb_depthwise_fwd_grouped", "yamb_depthwise_bwd_grouped",
                 "yamb_depthwise_grouped_grids"):
        assert name in nat.SYMBOLS and hasattr(built_lib, name)
    assert [f[0] for f in nat.DwFwdGrouped._fields_] == ["nbranch", "branch", "grid"]
    assert [f[0] for f in nat.DwBwdGrouped._fields_] == ["nbranch", "branch", "grid", "grid_wgrad"]


def test_predicate():
    """mb_dw_grouped on stand-in plans: the switch, an expansion and two or more branches."""
    import types
    from yet_another_mobilenet_series_b200 import engine
    ns = types.SimpleNamespace
    kind = ((3, 5, 7), 1, 56, 56, 24, (24, 8, 8))

    def plan(**kw):
        d = dict(expand=True, conv_dw=[0, 1, 2], mb_dw_kind=kind)
        d.update(kw)
        return ns(**d)
    old = (engine.TRAIN_MB_DW_GROUPED, engine.MB_DW_SHAPE_RULE)
    try:
        engine.MB_DW_SHAPE_RULE = False
        engine.TRAIN_MB_DW_GROUPED = False
        assert not engine.mb_dw_grouped(plan())
        engine.TRAIN_MB_DW_GROUPED = True
        assert engine.mb_dw_grouped(plan())
        assert engine.mb_dw_grouped(plan(conv_dw=[0, 1]))
        assert not engine.mb_dw_grouped(plan(conv_dw=[0]))
        assert not engine.mb_dw_grouped(plan(expand=False))
        engine.MB_DW_SHAPE_RULE = True
        assert engine.mb_dw_grouped(plan()) == (kind in engine.MB_DW_FASTER)
    finally:
        engine.TRAIN_MB_DW_GROUPED, engine.MB_DW_SHAPE_RULE = old
    fwd = inspect.getsource(engine.BlockPlan.forward)
    bwd = inspect.getsource(engine.BlockPlan.backward)
    assert "mb_dw_grouped(self) and self._dw_fwd_grouped()" in fwd
    assert "mb_dw_grouped(self) and not se_fused and self._dw_bwd_grouped(grads)" in bwd


def _multi_branch_blocks(model, hw):
    """(index, input H, block) of every block of model.features with several branches."""
    import torch
    from yet_another_mobilenet_series_b200 import engine
    out, H = [], hw
    for i, m in enumerate(model.features):
        if hasattr(m, "expand_conv") or hasattr(m, "ops"):
            if len(engine.block_parts(m).dws) > 1:
                out.append((i, H, m))
            H = (H - 1) // m.stride + 1
        else:
            for conv in [c for c in m.modules() if isinstance(c, torch.nn.Conv2d)][:1]:
                H = (H - 1) // conv.stride[0] + 1
    return out


def _check_plan(engine, m, H):
    plan = engine.mb_dw_group_plan(m, 2, H, H)
    parts = engine.block_parts(m)
    kind = engine.mb_dw_kind(m, H, H)
    assert kind == (tuple(br["k"] for br in plan), plan[0]["stride"], H, H,
                    parts.expand_convs[0].in_channels, tuple(br["C"] for br in plan))
    assert all(len(k) == 6 for k in engine.MB_DW_FASTER)
    assert plan is not None and len(plan) == len(parts.dws) <= 3
    c0 = 0
    for b, (br, (conv, _)) in enumerate(zip(plan, parts.dws)):
        # launch order = branch order of the module = channel order of the hidden tensor
        assert br["slot"] == b
        assert (br["k"], br["stride"]) == (conv.kernel_size[0], conv.stride[0])
        assert br["C"] == (conv.out_channels + 7) // 8 * 8 and br["c0"] == c0
        c0 += br["C"]
    assert len({br["stride"] for br in plan}) == 1
    assert c0 == sum((c + 7) // 8 * 8 for c in m.channels)
    return plan


@pytest.mark.parametrize("name", ["atomnas_a", "atomnas_a+", "atomnas_b", "atomnas_b+", "atomnas_c",
                                  "atomnas_c+"])
def test_group_plan_atomnas(flags_stub, name):
    """Every multi-branch block of the AtomNAS configurations is grouped: one slot per branch in
    the hidden tensor's channel order, with the (padded) channel slice of its statistics."""
    from yet_another_mobilenet_series_b200 import engine
    model, cfg = build_cfg(name)
    blocks = _multi_branch_blocks(model, cfg["flags"]["image_size"])
    assert blocks, name
    ks = set()
    for _i, H, m in blocks:
        plan = _check_plan(engine, m, H)
        ks |= {br["k"] for br in plan}
    assert ks == {3, 5, 7}
    # single-branch blocks keep their per-branch launch
    for m in model.features:
        if hasattr(m, "ops") and len(engine.block_parts(m).dws) == 1:
            assert engine.mb_dw_group_plan(m, 2, 56, 56) is None
            assert engine.mb_dw_kind(m, 56, 56) is None


def test_group_plan_supernet():
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    bn = {"momentum": 0.01, "eps": 1e-3}
    for stride in (1, 2):
        blk = mb.InvertedResidualChannels(24, 32, stride, [48, 48, 48], [3, 5, 7], True,
                                          mb.get_active_fn("nn.ReLU6"), bn)
        plan = _check_plan(engine, blk, 56)
        assert [(br["k"], br["c0"], br["C"]) for br in plan] == [(3, 0, 48), (5, 48, 48),
                                                                  (7, 96, 48)]
        assert {br["stride"] for br in plan} == {stride}


@pytest.fixture
def flags_stub(monkeypatch):
    import sys
    import types
    mod = types.ModuleType("utils.config")
    mod.FLAGS = types.SimpleNamespace()
    monkeypatch.setitem(sys.modules, "utils.config", mod)
    return mod


# ---- host validation ----------------------------------------------------------------------------
def _fwd_branch(nat, d, k, bn):
    d.N, d.H, d.W, d.C, d.ldc, d.k, d.stride = 2, 56, 56, 16, 48, k, 1
    d.x, d.y, d.w = 4096, 8192, 12288
    d.in_scale, d.in_shift, d.in_act = 16384, 20480, 2
    d.bn = C.pointer(bn)


def _fwd(nat, n=3):
    a = nat.DwFwdGrouped()
    a.nbranch = n
    bns = []
    for b in range(3):
        bn = nat.BnFwd()
        bn.partials, bn.counter, bn.scale, bn.shift, bn.count = 4096, 8192 + 4 * b, 12288, 16384, 2
        bns.append(bn)
        _fwd_branch(nat, a.branch[b], (3, 5, 7)[b], bn)
        a.grid[b] = 64
    return a, bns


def _bwd(nat, n=3):
    a = nat.DwBwdGrouped()
    a.nbranch = n
    bns = []
    for b in range(3):
        bn = nat.BnBwd()
        bn.partials, bn.counter, bn.count = 4096, 8192 + 4 * b, 2
        bns.append(bn)
        d = a.branch[b]
        d.N, d.H, d.W, d.C, d.ldc, d.k, d.stride = 2, 56, 56, 16, 48, (3, 5, 7)[b], 1
        d.dz, d.h, d.x, d.dx = 4096, 8192, 12288, 16384
        d.ca, d.cb, d.cc, d.w, d.dw = 20480, 24576, 28672, 32768, 36864
        d.in_scale, d.in_shift, d.in_act = 40960, 45056, 2
        d.bn = C.pointer(bn)
        a.grid[b] = 64
        a.grid_wgrad[b] = 64 if d.k == 7 else 0
    return a, bns


def test_refused_descriptors(built_lib):
    """Malformed descriptors: YAMB_EINVAL before any device work, with or without a device (the
    stand-in pointers are never used)."""
    from yet_another_mobilenet_series_b200 import native as nat
    lib = built_lib
    assert lib.yamb_depthwise_fwd_grouped(None, None) == -1
    assert lib.yamb_depthwise_bwd_grouped(None, None) == -1

    def fwd_case(edit):
        a, bns = _fwd(nat)
        edit(a, bns)
        return lib.yamb_depthwise_fwd_grouped(C.byref(a), None)

    def bwd_case(edit):
        a, bns = _bwd(nat)
        edit(a, bns)
        return lib.yamb_depthwise_bwd_grouped(C.byref(a), None)

    edits = [
        lambda a, b: setattr(a, "nbranch", 0),
        lambda a, b: setattr(a, "nbranch", 4),
        lambda a, b: setattr(a, "nbranch", -1),
        lambda a, b: a.grid.__setitem__(1, 0),
        lambda a, b: a.grid.__setitem__(2, -5),
        lambda a, b: a.grid.__setitem__(0, 2 ** 31 - 1) or a.grid.__setitem__(1, 2 ** 31 - 1),
        lambda a, b: setattr(a.branch[1], "stride", 2),            # strides differ
        lambda a, b: setattr(a.branch[2], "k", 4),
        lambda a, b: setattr(a.branch[0], "C", 12),                # not a multiple of 8
        lambda a, b: setattr(a.branch[1], "C", 56),                # C > ldc
        lambda a, b: setattr(a.branch[1], "C", 8192) or setattr(a.branch[1], "ldc", 8192),
        lambda a, b: setattr(a.branch[0], "N", 0),
        lambda a, b: setattr(b[1], "counter", b[0].counter),       # shared counter
    ]
    for i, e in enumerate(edits):
        assert fwd_case(e) == -1, i
        assert bwd_case(e) == -1, i
    # per-branch alignment and pointers
    for e in (lambda a, b: setattr(a.branch[1], "x", 4104), lambda a, b: setattr(a.branch[2], "y", 8200),
              lambda a, b: setattr(a.branch[0], "w", None)):
        assert fwd_case(e) == -1
    for e in (lambda a, b: setattr(a.branch[1], "dz", 4104), lambda a, b: setattr(a.branch[2], "dx", 16388),
              lambda a, b: setattr(a.branch[0], "dw", None),
              lambda a, b: a.grid_wgrad.__setitem__(2, 0),             # k = 7 needs both kernels
              lambda a, b: a.grid_wgrad.__setitem__(0, 8)):            # k = 3 has one
        assert bwd_case(e) == -1
    # the grid query runs the same checks
    a, _b = _fwd(nat)
    a.branch[1].stride = 2
    assert lib.yamb_depthwise_grouped_grids(C.byref(a), None) == -1


def test_no_device(built_lib):
    """Valid descriptors without a device: YAMB_ENODEV from the launchers and the grid query."""
    import torch
    from yet_another_mobilenet_series_b200 import native as nat
    if torch.cuda.is_available():
        pytest.skip("checks the answer without a device")
    for n in (1, 2, 3):
        a, _b = _fwd(nat, n)
        assert built_lib.yamb_depthwise_fwd_grouped(C.byref(a), None) == -2
        assert built_lib.yamb_depthwise_grouped_grids(C.byref(a), None) == -2
        g, _c = _bwd(nat, n)
        assert built_lib.yamb_depthwise_bwd_grouped(C.byref(g), None) == -2
        assert built_lib.yamb_depthwise_grouped_grids(None, C.byref(g)) == -2
