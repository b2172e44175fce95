"""CPU: the drop-in boundary — module surface of models/mobilenet_base.py, builders, C-ABI library
exports.  Mirrors the reference's own structural tests (tests/models/mobilenet_base_test.py)."""
import ctypes
import os
import re

import pytest
import torch
from torch import nn

from yet_another_mobilenet_series_b200 import mobilenet_base as mb
from yet_another_mobilenet_series_b200 import mobilenet_supernet, searched_network

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BN = {"momentum": 0.01, "eps": 1e-3}


def _unfused(expand=True):
    if expand:
        return mb.InvertedResidualChannels(16, 24, 1, [48, 32], [3, 5], True,
                                           mb.get_active_fn("nn.ReLU6"), BN)
    return mb.InvertedResidualChannels(16, 24, 1, [16], [3], False, mb.get_active_fn("nn.ReLU"), BN)


def _fused():
    return mb.InvertedResidualChannelsFused(16, 16, 1, [48, 32], [3, 5], True,
                                            mb.get_active_fn("nn.Swish"), BN, se_ratio=0.5)


def test_get_named_depthwise_bn_keys_and_types():
    # reference tests/models/mobilenet_base_test.py:15-35, 44-64
    for blk, fmt in ((_unfused(), "ops.{}.1.1"), (_unfused(False), "ops.{}.0.1"),
                     (_fused(), "depth_ops.{}.1.1")):
        named = blk.get_named_depthwise_bn()
        assert list(named) == [fmt.format(i) for i in range(len(blk.channels))]
        assert all(isinstance(v, nn.BatchNorm2d) for v in blk.get_depthwise_bn())
        pref = blk.get_named_depthwise_bn(prefix="features.3")
        assert list(pref) == ["features.3." + k for k in named]
        mods = dict(blk.named_modules())
        assert all(mods[k] is v for k, v in named.items())


def test_state_dict_layout():
    sd = _unfused().state_dict()
    assert sd["ops.0.0.0.weight"].shape == (48, 16, 1, 1)
    assert sd["ops.1.1.0.weight"].shape == (32, 1, 5, 5)
    assert sd["ops.1.2.weight"].shape == (24, 32, 1, 1)
    assert "pw_bn.num_batches_tracked" in sd
    sd = _unfused(False).state_dict()
    assert sd["ops.0.0.0.weight"].shape == (16, 1, 3, 3) and sd["ops.0.1.weight"].shape == (24, 16, 1, 1)
    sd = _fused().state_dict()
    assert sd["expand_conv.0.weight"].shape == (80, 16, 1, 1)
    assert sd["depth_ops.1.1.0.weight"].shape == (32, 1, 5, 5)
    assert sd["project_conv.0.weight"].shape == (16, 80, 1, 1)
    assert sd["se_op.se_reduce.weight"].shape == (8, 80, 1, 1)  # round(inp * se_ratio)
    assert sd["se_op.se_expand.bias"].shape == (80,)


def test_ctor_errors_and_attributes():
    with pytest.raises(AssertionError):
        mb.InvertedResidualChannels(16, 16, 3, [16], [3], True, mb.get_active_fn("nn.ReLU"))
    with pytest.raises(AssertionError):
        mb.InvertedResidualChannels(16, 16, 1, [16, 16], [3], True, mb.get_active_fn("nn.ReLU"))
    with pytest.raises(RuntimeError):
        mb.InvertedResidualChannels(16, 16, 1, [32], [3], False, mb.get_active_fn("nn.ReLU"))
    blk = _unfused()
    assert (blk.input_dim, blk.output_dim, blk.stride, blk.expand) == (16, 24, 1, True)
    assert not blk.use_res_connect and _fused().use_res_connect
    assert repr(blk).startswith("InvertedResidualChannels(16, 24, channels=[48, 32], "
                                "kernel_sizes=[3, 5], expand=True, stride=1)")
    assert "se_ratio=0.5, nl_s=0, nl_c=0" in repr(_fused())


def test_registries_and_activations():
    assert mb.get_block("InvertedResidualChannels") is mb.InvertedResidualChannels
    assert mb.get_block("InvertedResidualChannelsFused") is mb.InvertedResidualChannelsFused
    x = torch.linspace(-5, 8, 27)
    assert torch.equal(mb.get_active_fn("nn.ReLU6")()(x.clone()), x.clamp(0, 6))
    assert torch.allclose(mb.get_active_fn("nn.Swish")()(x), x * torch.sigmoid(x))
    assert torch.allclose(mb.get_active_fn("nn.HSwish")()(x), x * (x + 3).clamp(0, 6) / 6)
    assert isinstance(mb.get_active_fn("nn.HSwish")(), nn.Module)  # usable in nn.Sequential
    assert mb._make_divisible(32 * 0.35, 8) == 16 and mb._make_divisible(10, 8) == 16


def test_mobilenet_v2_builder_param_count_and_deepcopy():
    import copy
    rows = [[1, 16, 1, 1, [3]], [6, 24, 2, 2, [3]], [6, 32, 3, 2, [3]], [6, 64, 4, 2, [3]],
            [6, 96, 3, 1, [3]], [6, 160, 3, 2, [3]], [6, 320, 1, 1, [3]]]
    m = mobilenet_supernet.Model(inverted_residual_setting=rows, active_fn="nn.ReLU",
                                 batch_norm_momentum=0.01, batch_norm_epsilon=1e-3, input_size=224)
    assert sum(p.numel() for p in m.parameters()) == 3504872  # SURVEY.md §6 cross-check
    assert len(list(m.parameters())) == 158
    m2 = copy.deepcopy(m)  # get_ema_model deep-copies the model (reference common.py:164)
    assert m2.features[3].ops[0][0][0].weight is not m.features[3].ops[0][0][0].weight
    with pytest.raises(ValueError):
        mobilenet_supernet.Model(inverted_residual_setting=rows, input_size=200)
    with pytest.raises(ValueError):
        mobilenet_supernet.Model(inverted_residual_setting=[[1, 2, 3]], input_size=224)


def test_searched_builder():
    rows = [[16, 1, 1, [3], [32], False], [24, 2, 2, [3, 5], [48, 24], True]]
    m = searched_network.Model(inverted_residual_setting=rows, input_size=224,
                               block="InvertedResidualChannelsFused", se_ratio=0.5,
                               active_fn="nn.Swish")
    assert isinstance(m.features[2], mb.InvertedResidualChannelsFused)
    assert m.features[2].se_op.n_hidden == 8
    with pytest.raises(NotImplementedError):
        searched_network.Model(inverted_residual_setting=rows, input_size=224, se_ratio=0.5)
    with pytest.raises(ValueError):
        searched_network.Model(inverted_residual_setting=rows, input_size=224, width_mult=0.5)


def test_capi_exports_every_declared_symbol(built_lib):
    """The C-ABI library loads without a GPU and exports every function include/yamb200.h
    declares; struct sizes agree with the ctypes mirror (checked inside native.lib())."""
    from yet_another_mobilenet_series_b200 import native
    hdr = open(os.path.join(ROOT, "include", "yamb200.h")).read()
    declared = set(re.findall(r"\b(yamb_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(native.SYMBOLS)
    raw = ctypes.CDLL(native.LIB_PATH)
    for sym in declared:
        assert hasattr(raw, sym), sym
    assert built_lib.yamb_version() >= 100


def test_no_cpu_fallback(built_lib):
    """Compute entry points refuse to run without a device; the block refuses CPU tensors."""
    from yet_another_mobilenet_series_b200 import native
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    g = native.Gemm()
    g.M = g.N = g.K = 64
    rc = built_lib.yamb_pointwise_gemm(ctypes.byref(g), None)
    assert rc == -2 and b"no CUDA device" in built_lib.yamb_last_error()
    with pytest.raises(native.NativeError):
        _unfused()(torch.randn(2, 16, 8, 8))


def test_fused_rmsprop_ctor_contract():
    from yet_another_mobilenet_series_b200.fused_rmsprop import RMSprop, mnas_l2_mask
    p = [nn.Parameter(torch.zeros(3))]
    for kw in (dict(lr=-1), dict(eps=-1), dict(momentum=-1), dict(weight_decay=-1), dict(alpha=-1)):
        with pytest.raises(ValueError):
            RMSprop(p, **kw)
    opt = RMSprop(p, lr=0.016, alpha=0.9, momentum=0.9, eps=1e-3, eps_inside_sqrt=True)
    assert opt.param_groups[0]["eps_inside_sqrt"] is True and opt.defaults["centered"] is False
    m = nn.Sequential()
    m.add_module("conv", nn.Conv2d(4, 8, 1, bias=False))
    m.add_module("bn", nn.BatchNorm2d(8))
    m.add_module("classifier", nn.Linear(8, 5))
    assert mnas_l2_mask(m.named_parameters()) == {
        "conv.weight": True, "bn.weight": False, "bn.bias": False, "classifier.weight": True,
        "classifier.bias": True}


def test_padded_shadow_flat_transfers_cpu():
    """AtomNAS-style odd widths: the zero-padded shadow block's batched transfers (one gather each
    way, engine._PadShadow) put every real value where the per-tensor maps say, pads are 0 (1 for a
    running variance), and the gradient gather is the exact inverse."""
    from yet_another_mobilenet_series_b200 import engine
    torch.manual_seed(0)
    blk = mb.InvertedResidualChannelsFused(24, 24, 1, [15, 23, 13], [3, 5, 7], True,
                                           mb.get_active_fn("nn.Swish"), BN, se_ratio=0.5)
    for p in blk.parameters():
        p.data.normal_()
    for n, b in blk.named_buffers():
        if b.dim():
            b.data.uniform_(0.5, 2.0)
    sh = engine._PadShadow(blk, torch.device("cpu"))
    sh.push(blk)
    real = dict(blk.named_parameters())
    real.update(dict(blk.named_buffers()))
    shad = dict(sh.shadow.named_parameters())
    shad.update(dict(sh.shadow.named_buffers()))
    for name, t in real.items():
        st = shad[name]
        if t.dim() == 0:
            assert int(st) == int(t)
            continue
        m = sh.maps[name]
        assert torch.equal(st.reshape(-1)[m], t.reshape(-1)), name
        mask = torch.ones(st.numel(), dtype=torch.bool)
        mask[m] = False
        pad = st.reshape(-1)[mask]
        want = 1.0 if name.endswith("running_var") else 0.0
        assert bool((pad == want).all()), name
    # statistics come back; gradients gather to the real shapes
    for n in sh.stat_names:
        shad[n].add_(1.0)
    before = {n: real[n].clone() for n in sh.stat_names}
    sh.pull_stats(blk)
    for n in sh.stat_names:
        assert torch.allclose(real[n], before[n] + 1.0), n
    sp = dict(sh.shadow.named_parameters())
    gmap = {id(p): torch.arange(p.numel(), dtype=torch.float32).view(p.shape) for p in sp.values()}
    grads = sh.gather_grads(gmap, blk)
    for (n, p), g in zip(blk.named_parameters(), grads):
        assert g.shape == p.shape
        assert torch.equal(g.reshape(-1), sh.maps[n].float()), n


def test_grad_targets_split_concatenated_weight_gradients_cpu():
    """engine.GradTargets: a multi-branch project weight gradient is one [Cout, Chid] buffer whose
    column slices become the branch weights' gradients; in direct mode they are added into the
    `.grad` views and the buffer is kept by its owner, in autograd mode they are returned."""
    from yet_another_mobilenet_series_b200 import engine
    ws = [nn.Parameter(torch.zeros(8, c, 1, 1)) for c in (3, 5)]
    full = torch.arange(64, dtype=torch.float32).view(8, 8)
    owner = {}
    for direct in (False, True):
        for w in ws:
            w.grad = torch.ones_like(w) if direct else None
            w._yamb_direct = direct
        gt = engine.GradTargets(ws)
        assert gt.direct == direct and gt.host_reads != direct
        buf = gt.concat(ws, 1, owner, "proj")
        assert gt.host_reads                       # the split reads the buffer after the kernels
        assert buf.shape == (8, 8) and bool((buf == 0).all())
        assert ("proj" in owner) == direct
        buf.copy_(full)
        got = gt.result()
        want = [full[:, :3].reshape(8, 3, 1, 1), full[:, 3:].reshape(8, 5, 1, 1)]
        if direct:
            assert got == (None, None)
            got = [w.grad - 1 for w in ws]
        for g, t in zip(got, want):
            assert torch.equal(g, t)
    single = engine.GradTargets(ws[:1])            # direct, one branch: the `.grad` itself
    assert single.concat(ws[:1], 1, owner, "x").data_ptr() == ws[0].grad.data_ptr()
    assert not single.host_reads and "x" not in owner
    ws[1]._yamb_direct = False                     # mixed ownership: autograd mode
    assert not engine.GradTargets(ws).direct


def test_kernel_scratch_does_not_travel_with_a_deepcopy():
    """The EMA model is a deepcopy of the wrapper (reference common.py:164), possibly taken AFTER a
    forward has cached per-module kernel scratch (device buffers, ctypes argument structs) in the
    modules' __dict__: the copy must succeed and start without scratch."""
    import copy
    import pickle
    from yet_another_mobilenet_series_b200 import engine, native, tail_ops

    class Holder(engine.Scratch):
        def __init__(self):
            self.arg = native.Gemm()          # ctypes struct with pointers: not copyable

    blk = mb.InvertedResidualChannels(16, 16, 1, [32], [3], True, active_fn=mb.get_active_fn("nn.ReLU"),
                                      batch_norm_kwargs={"momentum": 0.01, "eps": 1e-3})
    head = mb.ConvBNReLU(16, 32, kernel_size=1, active_fn=mb.get_active_fn("nn.ReLU"))
    seq = nn.Sequential(blk, nn.Linear(4, 4), head)
    plans = engine._ScratchDict()
    plans["k"] = Holder()
    blk.__dict__["_yamb_plans"] = plans
    blk.__dict__["_yamb_eval"] = engine._ScratchDict(a=torch.zeros(1))
    blk.pw_bn.__dict__["_yamb_bnact"] = Holder()
    seq[1].__dict__["_yamb_lin"] = Holder()
    head[0].__dict__["_yamb_pw"] = Holder()
    assert issubclass(tail_ops._PwState, engine.Scratch)
    assert issubclass(tail_ops._LinearState, engine.Scratch)
    assert issubclass(engine._BnActState, engine.Scratch)
    c = copy.deepcopy(seq)
    assert "_yamb_plans" not in c[0].__dict__ and "_yamb_eval" not in c[0].__dict__
    assert c[0].pw_bn.__dict__["_yamb_bnact"] is None and c[1].__dict__["_yamb_lin"] is None
    assert c[2][0].__dict__["_yamb_pw"] is None
    for (k, a), (_, b) in zip(seq.state_dict().items(), c.state_dict().items()):
        assert torch.equal(a, b), k
    r = pickle.loads(pickle.dumps(seq[1]))
    assert r.__dict__["_yamb_lin"] is None
    r = pickle.loads(pickle.dumps(head))
    assert r[0].__dict__["_yamb_pw"] is None


def test_one_launch_eval_dispatch_rules():
    """engine.eval_supported decides from module structure only (no GPU needed): eval + no_grad +
    single-branch k in {3,5,7}; everything else keeps the four-launch path."""
    from yet_another_mobilenet_series_b200 import engine
    bn = {"momentum": 0.01, "eps": 1e-3}
    relu, swish = mb.get_active_fn("nn.ReLU6"), mb.get_active_fn("nn.Swish")
    x = torch.zeros(2, 32, 14, 14)

    def blk(*a, **k):
        return mb.InvertedResidualChannels(*a, **k).eval()

    plain = blk(32, 32, 1, [192], [3], True, active_fn=relu, batch_norm_kwargs=bn)
    assert not engine.eval_supported(plain, x)              # gradient mode is on
    with torch.no_grad():
        assert engine.eval_supported(plain, x)
        assert engine.eval_supported(blk(32, 64, 2, [192], [7], True, active_fn=relu,
                                         batch_norm_kwargs=bn), x)
        assert engine.eval_supported(blk(32, 16, 1, [32], [3], False, active_fn=relu,
                                         batch_norm_kwargs=bn), x)
        assert engine.eval_supported(blk(32, 32, 1, [96], [3], True, active_fn=swish,
                                         batch_norm_kwargs=bn), x)
        # not covered: Swish with k = 5, several branches, odd widths, train mode
        assert not engine.eval_supported(blk(32, 32, 1, [96], [5], True, active_fn=swish,
                                             batch_norm_kwargs=bn), x)
        assert not engine.eval_supported(blk(32, 32, 1, [48, 48], [3, 5], True, active_fn=relu,
                                             batch_norm_kwargs=bn), x)
        assert not engine.eval_supported(blk(32, 32, 1, [90], [3], True, active_fn=relu,
                                             batch_norm_kwargs=bn), x)
        fused = mb.InvertedResidualChannelsFused(32, 32, 1, [96], [3], True, active_fn=relu,
                                                 batch_norm_kwargs=bn).eval()
        assert engine.eval_supported(fused, x)              # the fused class's rule
        assert not engine.eval_supported(plain.train(), x)
        plain.eval()
        prev, engine.EVAL_FUSED = engine.EVAL_FUSED, False
        try:
            assert not engine.eval_supported(plain, x)      # YAMB_EVAL_FUSED=0
        finally:
            engine.EVAL_FUSED = prev


@pytest.mark.parametrize("make,paths", [
    (lambda: _unfused(True),
     (["ops.0.0.0", "ops.1.0.0"], ["ops.0.0.1", "ops.1.0.1"],
      [("ops.0.1.0", "ops.0.1.1"), ("ops.1.1.0", "ops.1.1.1")], ["ops.0.2", "ops.1.2"], "pw_bn",
      None, None)),
    (lambda: _unfused(False),
     ([], [], [("ops.0.0.0", "ops.0.0.1")], ["ops.0.1"], "pw_bn", None, None)),
    (lambda: mb.InvertedResidualChannelsFused(16, 16, 1, [48, 32], [3, 5], True,
                                              mb.get_active_fn("nn.Swish"), BN, se_ratio=0.5,
                                              nl_c=0.25, nl_s=1),
     (["expand_conv.0"], ["expand_conv.1"],
      [("depth_ops.0.1.0", "depth_ops.0.1.1"), ("depth_ops.1.1.0", "depth_ops.1.1.1")],
      ["project_conv.0"], "project_conv.1", "se_op", "nl_op")),
    (lambda: mb.InvertedResidualChannelsFused(16, 24, 1, [16], [3], False,
                                              mb.get_active_fn("nn.ReLU"), BN, nl_c=0.25, nl_s=1),
     ([], [], [("depth_ops.0.0.0", "depth_ops.0.0.1")], ["project_conv.0"], "project_conv.1",
      None, "nl_op")),
], ids=["unfused_expand_2branch", "unfused_no_expand", "fused_expand_2branch_se_nl",
        "fused_no_expand_nl"])
def test_block_parts_follow_the_reference_module_tree(make, paths):
    """engine.block_parts returns, for either block class, the modules at the reference's
    state_dict paths."""
    from yet_another_mobilenet_series_b200 import engine
    blk = make()
    keys = set(blk.state_dict())
    exp, bn1, dws, proj, bn3, se, nl = paths

    def at(path):
        assert any(k.startswith(path + ".") for k in keys), path
        return blk.get_submodule(path)

    p = engine.block_parts(blk)
    assert p.fused == isinstance(blk, mb.InvertedResidualChannelsFused)
    assert [id(m) for m in p.expand_convs] == [id(at(q)) for q in exp]
    assert [id(m) for m in p.bn1s] == [id(at(q)) for q in bn1]
    assert [(id(c), id(b)) for c, b in p.dws] == [(id(at(c)), id(at(b))) for c, b in dws]
    assert [id(m) for m in p.project_convs] == [id(at(q)) for q in proj]
    assert p.bn3 is at(bn3)
    assert p.se is (None if se is None else at(se))
    assert p.nl is (None if nl is None else at(nl))
    assert isinstance(p.bn3, nn.BatchNorm2d) and all(isinstance(b, nn.BatchNorm2d) for b in p.bn1s)
