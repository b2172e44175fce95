"""CPU: the training-mode expand + depthwise forward from x (TrainStep(fused_expand_dw=True)): the
ABI struct mirror, refused arguments and the answer without a device, which blocks of the four
configurations the dispatch and the shape rule select, and that the switch is off outside a step."""
import ctypes as C
import inspect
import sys
import types

import pytest


@pytest.fixture
def flags(monkeypatch):
    """A stand-in for the reference's utils.config (the non-local block reads FLAGS)."""
    mod = types.ModuleType("utils.config")
    mod.FLAGS = types.SimpleNamespace()
    monkeypatch.setitem(sys.modules, "utils.config", mod)
    return mod


def test_switch_off_by_default():
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    assert engine.TRAIN_EXPAND_DW_FUSED is False
    assert inspect.signature(TrainStep).parameters["fused_expand_dw"].default is False


def test_switch_set_only_inside_the_step():
    """TrainStep sets the switch in _fwd_bwd (eager, captured and micro-batched passes all run
    through it) and clears it in the `finally` of the same call; it is not a checkpoint field."""
    from yet_another_mobilenet_series_b200 import trainer
    src = inspect.getsource(trainer.TrainStep._fwd_bwd)
    on = src.index("engine.TRAIN_EXPAND_DW_FUSED = self.fused_expand_dw")
    fin = src.index("finally:")
    assert on < src.index("self._passes(") < fin
    assert "engine.TRAIN_EXPAND_DW_FUSED = False" in src[fin:]
    whole = inspect.getsource(trainer)
    assert whole.count("engine.TRAIN_EXPAND_DW_FUSED =") == 2
    for fn in ("state_dict", "load_state_dict", "save_status"):
        if hasattr(trainer.TrainStep, fn):
            assert "fused_expand_dw" not in inspect.getsource(getattr(trainer.TrainStep, fn))


def test_struct_size(built_lib):
    from yet_another_mobilenet_series_b200 import native as nat
    assert built_lib.yamb_struct_size(40) == C.sizeof(nat.ExpandDwTrain)
    assert "yamb_expand_dw_train_fwd" in nat.SYMBOLS and hasattr(built_lib, "yamb_expand_dw_train_fwd")
    names = [f[0] for f in nat.ExpandDwTrain._fields_]
    assert names == ["N", "H", "W", "Cin", "Chid", "kernel", "stride", "act", "ldh", "x",
                     "w_expand", "bn1_scale", "bn1_shift", "w_dw", "h2", "bn"]


def _args(nat, bn=None, **kw):
    bn = bn or nat.BnFwd()
    bn.partials, bn.counter, bn.scale, bn.shift, bn.count = 4096, 8192, 12288, 16384, 2 * 56 * 56
    a = nat.ExpandDwTrain()
    a.N, a.H, a.W, a.Cin, a.Chid, a.kernel, a.stride, a.act, a.ldh = 2, 56, 56, 24, 144, 3, 1, 2, 144
    a.x, a.w_expand, a.bn1_scale, a.bn1_shift, a.w_dw, a.h2 = (4096 * i for i in range(10, 16))
    a.bn = C.pointer(bn)
    for k, v in kw.items():
        if k.startswith("bn_"):
            setattr(bn, k[3:], v)
        else:
            setattr(a, k, v)
    return a, bn


def test_no_device(built_lib):
    """Valid arguments without a device: YAMB_ENODEV, for every (k, stride) and channel counts up
    to the caps."""
    import torch
    from yet_another_mobilenet_series_b200 import native as nat
    if torch.cuda.is_available():
        pytest.skip("checks the answer without a device")
    for k in (3, 5, 7):
        for s in (1, 2):
            for cin, chid in ((8, 8), (24, 144), (256, 1536), (160, 960)):
                for act in range(5):
                    a, _bn = _args(nat, kernel=k, stride=s, Cin=cin, Chid=chid, ldh=chid, act=act)
                    assert built_lib.yamb_expand_dw_train_fwd(C.byref(a), None) == -2, (k, s, cin)


def test_refused_arguments(built_lib):
    """Shapes the kernel does not cover and malformed arguments: YAMB_EINVAL, with or without a
    device (every check comes before the device query, so the stand-in pointers are never used)."""
    from yet_another_mobilenet_series_b200 import native as nat
    lib = built_lib
    for kw in ({"N": 0}, {"H": 0}, {"W": -1}, {"Cin": 0}, {"Cin": 12}, {"Cin": 264},
               {"Chid": 0}, {"Chid": 100}, {"kernel": 4}, {"kernel": 1}, {"kernel": 9},
               {"stride": 3}, {"stride": 0}, {"act": 5}, {"act": -1}, {"ldh": 136}, {"ldh": 148},
               {"x": None}, {"w_expand": None}, {"bn1_scale": None}, {"bn1_shift": None},
               {"w_dw": None}, {"h2": None}, {"x": 4104}, {"w_expand": 4100}, {"h2": 4104},
               {"bn_partials": None}, {"bn_counter": None}, {"bn_scale": None},
               {"bn_shift": None}, {"N": 65536, "H": 256, "W": 256}):
        a, _bn = _args(nat, **kw)
        assert lib.yamb_expand_dw_train_fwd(C.byref(a), None) == -1, kw
    a, _bn = _args(nat)
    a.bn = None
    assert lib.yamb_expand_dw_train_fwd(C.byref(a), None) == -1
    assert lib.yamb_expand_dw_train_fwd(None, None) == -1


def _shapes(model, hw):
    """Input H (= W) of every block of model.features: the stem and each block's stride."""
    import torch
    out, H = {}, hw
    for i, m in enumerate(model.features):
        if hasattr(m, "expand_conv") or hasattr(m, "ops"):
            out[i] = H
            H = (H - 1) // m.stride + 1
        else:
            for conv in [c for c in m.modules() if isinstance(c, torch.nn.Conv2d)][:1]:
                H = (H - 1) // conv.stride[0] + 1
    return out


# covered blocks: single branch with expansion; MobileNetV2 / Proxyless / AutoNL-L have one branch
# everywhere, so every block but the first (no expansion); AtomNAS-C+ has no single-branch block
# with expansion
EXPECT = {"mobilenet_v2": (17, 16), "proxyless_mobile": (20, None), "autonl_l": (None, None),
          "atomnas_c+": (None, 0)}


@pytest.mark.parametrize("name", ["mobilenet_v2", "proxyless_mobile", "autonl_l", "atomnas_c+"])
def test_dispatch_and_shape_rule(flags, monkeypatch, name):
    """Which blocks the dispatch covers (one branch, an expansion) and which of those the shape
    rule sends down the path, through the predicate BlockPlan.forward uses."""
    from _cfg import build_from_cfg
    from yet_another_mobilenet_series_b200 import engine
    assert "expand_dw_fused(self)" in inspect.getsource(engine.BlockPlan.forward)
    assert "_expand_dw_rule(plan.expand_dw_kind)" in inspect.getsource(engine.expand_dw_fused)
    model, cfg = build_from_cfg(name)
    shapes = _shapes(model, cfg["flags"]["image_size"])
    assert shapes
    covered = {}
    for i, H in shapes.items():
        m = model.features[i]
        parts = engine.block_parts(m)
        kind = engine.expand_dw_kind(m, H, H)
        want = bool(parts.expand_convs) and len(parts.dws) == 1
        assert (kind is not None) == want, (i, kind)
        if kind is not None:
            k, s, h, w, cin, chid = kind
            conv = parts.dws[0][0]
            assert (k, s, h, w) == (conv.kernel_size[0], conv.stride[0], H, H)
            assert (cin, chid) == (m.input_dim if hasattr(m, "input_dim") else cin, sum(m.channels))
            covered[i] = kind
    n_blocks, n_cov = EXPECT[name]
    if n_blocks is not None:
        assert len(shapes) == n_blocks, len(shapes)
    if n_cov is not None:
        assert len(covered) == n_cov, len(covered)
    if name != "atomnas_c+":
        assert len(covered) == len(shapes) - 1   # block 1 has no expansion
    # the shape rule: only kinds in EXPAND_DW_FASTER, or every covered block when it is off
    for i, H in shapes.items():
        m = model.features[i]
        assert engine.expand_dw_selected(m, H, H) == (covered.get(i) in engine.EXPAND_DW_FASTER)
    monkeypatch.setattr(engine, "EXPAND_DW_SHAPE_RULE", False)
    for i, H in shapes.items():
        assert engine.expand_dw_selected(model.features[i], H, H) == (i in covered)
    # every kind the rule lists is one these configurations have at the bench input size
    kinds = set(covered.values())
    assert all(len(k) == 6 for k in engine.EXPAND_DW_FASTER)
    if name == "mobilenet_v2":
        assert {k for k in engine.EXPAND_DW_FASTER if k[4:] == (16, 96)} <= kinds


def test_predicate_needs_switch_training_and_one_branch():
    """expand_dw_fused on stand-in plans: the switch, an expansion, one branch and batch
    statistics in both BatchNorms are all required."""
    from yet_another_mobilenet_series_b200 import engine
    ns = types.SimpleNamespace
    kind = (3, 1, 56, 56, 24, 144)

    def plan(**kw):
        d = dict(expand=True, conv_dw=[object()], bn1=ns(batch_stats=True),
                 bn2=ns(batch_stats=True), expand_dw_kind=kind)
        d.update(kw)
        return ns(**d)
    old = (engine.TRAIN_EXPAND_DW_FUSED, engine.EXPAND_DW_SHAPE_RULE)
    try:
        engine.EXPAND_DW_SHAPE_RULE = False
        engine.TRAIN_EXPAND_DW_FUSED = False
        assert not engine.expand_dw_fused(plan())
        engine.TRAIN_EXPAND_DW_FUSED = True
        assert engine.expand_dw_fused(plan())
        assert not engine.expand_dw_fused(plan(expand=False, bn1=None))
        assert not engine.expand_dw_fused(plan(conv_dw=[object(), object()]))
        assert not engine.expand_dw_fused(plan(bn1=ns(batch_stats=False)))
        assert not engine.expand_dw_fused(plan(bn2=ns(batch_stats=False)))
        assert not engine.expand_dw_fused(plan(expand_dw_kind=None))
        engine.EXPAND_DW_SHAPE_RULE = True
        assert engine.expand_dw_fused(plan()) == (kind in engine.EXPAND_DW_FASTER)
    finally:
        engine.TRAIN_EXPAND_DW_FUSED, engine.EXPAND_DW_SHAPE_RULE = old
