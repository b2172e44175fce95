"""Small-batch eval of the searched networks on the GPU: the multi-branch block kernel split over a
thread-block cluster (yamb_block_eval_mb_cluster_fwd / _pool_fwd) and EvalStep(small_batch=True).
  * every new instantiation (tile geometry x lean / generic activation x plain / gate / pool, at
    cluster sizes 2, 4 and 8) through the C ABI, element by element against the fp64 intervals of
    tests/block_eval_ref64.py per 64-channel slice, on the multi-tile and single-tile walks of
    tests/test_block_eval_mb_gpu.py; the same bits on a second run; the pool pass bitwise the
    unsplit one, the block output within fp32 reassociation of it;
  * a tile plan whose partials do not fit shared memory runs the unsplit launch;
  * every multi-branch block of AtomNAS-C / C+ at N = 1 through the engine, against fp32 truth
    with the autocast yardstick;
  * whole AtomNAS-C, C+ and AutoNL-L EvalStep(small_batch=True) logits at N = 1, 2 and 8 against
    fp32 truth and the default EvalStep, within the yardstick; the default EvalStep is unchanged by
    the table and the switch."""
import copy
import ctypes as C

import pytest
import torch

from test_block_eval_mb_gpu import CASES, _args, _case_tensors, _reference
from test_block_eval_mb_cpu import multi_branch_blocks

pytestmark = pytest.mark.gpu
DEV = "cuda"
SLACK, FLOOR = 1.5, 2.5e-3


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _call(lib, m, mode, cs, N, Ho, Cout, Chid):
    """One call of the split (cs > 1) or unsplit (cs = 1) entry point into a guarded buffer:
    (return code, output)."""
    from yet_another_mobilenet_series_b200 import native as nat
    st = nat.stream_handle()
    if mode == "pool":
        out = torch.full((N * Chid + 8,), 7.0, device=DEV)
        m.base.pooled = out.data_ptr()
        rc = lib.yamb_block_eval_mb_pool_fwd(C.byref(m), st) if cs == 1 else \
            lib.yamb_block_eval_mb_cluster_pool_fwd(C.byref(m), cs, st)
    else:
        out = torch.full((N * Ho * Ho * Cout + 8,), 7.0, device=DEV, dtype=torch.bfloat16)
        m.base.y = out.data_ptr()
        rc = lib.yamb_block_eval_mb_fwd(C.byref(m), st) if cs == 1 else \
            lib.yamb_block_eval_mb_cluster_fwd(C.byref(m), cs, st)
    torch.cuda.synchronize()
    if rc == 0:
        assert (out[-8:].float() == 7.0).all(), "guard values overwritten"
    return rc, out[:-8]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "k%d_s%d_n%d_h%d_co%d" % (c[:4] + (c[5],)))
@pytest.mark.parametrize("act", [1, 3], ids=["relu", "swish"])
@pytest.mark.parametrize("cs", [2, 4, 8])
def test_instantiations_against_fp64(built_lib, case, act, cs):
    from yet_another_mobilenet_series_b200 import native as nat
    K, S, N, H, Cin, Cout, groups = case
    Ho = (H - 1) // S + 1
    for mode, seed in (("plain", 1), ("gate", 2), ("pool", 3)):
        t = _case_tensors(case, act, seed + 10 * act)
        residual = mode == "plain" and S == 1 and Cin == Cout
        m = _args(case, t, act, mode, residual)
        rc, got = _call(built_lib, m, mode, cs, N, Ho, Cout, t["Chid"])
        nat.check(rc)
        rc, again = _call(built_lib, m, mode, cs, N, Ho, Cout, t["Chid"])
        assert torch.equal(got, again), "two runs differ"
        _, unsplit = _call(built_lib, m, mode, 1, N, Ho, Cout, t["Chid"])
        if mode == "pool":
            assert torch.equal(got, unsplit)          # each rank pools its own slices
            got = got.view(N, t["Chid"]).double()
        else:
            assert _rel(got.float(), unsplit.float()) < 1e-2, (mode, _rel(got.float(), unsplit.float()))
            got = got.view(N, Ho, Ho, Cout).permute(0, 3, 1, 2).double()
        lo, hi = _reference(case, t, act, mode, residual)
        bad = ~((got >= lo) & (got <= hi))
        assert not bad.any(), (mode, int(bad.sum()), got[bad][:4], lo[bad][:4], hi[bad][:4])


def test_no_fit_falls_back_to_the_unsplit_launch(built_lib, monkeypatch):
    """K_MAX 7 at stride 1 with Cin = 128 and Cout = 320: the tile plan fits shared memory, the
    cluster's exchanged partials do not.  The entry point declines with nothing enqueued and the
    engine runs the unsplit kernel (the same bits)."""
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    torch.manual_seed(0)
    blk = mb.InvertedResidualChannels(128, 320, 1, [256, 200], [7, 3], True, mb.get_active_fn("nn.ReLU"),
                                      {"momentum": 0.01, "eps": 1e-3}).to(DEV).eval()
    x = engine.to_nhwc_bf16(torch.randn(1, 128, 7, 7, device=DEV))
    monkeypatch.setattr(engine, "EVAL_SMALL_BATCH", True)
    monkeypatch.setattr(engine, "SMALL_BATCH_RULE", False)
    monkeypatch.setattr(engine, "EVAL_CLUSTER", 2)
    c0, l0 = engine.EVAL_MB_CLUSTER_CALLS, engine.LAUNCHES
    with torch.no_grad():
        y = blk(x)
    torch.cuda.synchronize()
    assert engine.EVAL_MB_CLUSTER_CALLS == c0 and engine.LAUNCHES == l0 + 2   # pack + unsplit
    assert b"shared memory" in built_lib.yamb_last_error()
    monkeypatch.setattr(engine, "EVAL_CLUSTER", 1)
    with torch.no_grad():
        assert torch.equal(y, blk(x))


# ---- modules and networks ----------------------------------------------------------------------
_NETS = {}


def _net(name):
    """The network with non-zero ZeroInitBN gammas and SE biases, its BatchNorm statistics
    calibrated on random images by the stock-torch graph."""
    import test_block_eval_mb_gpu
    import test_fused_class_eval_gpu
    if name not in _NETS:
        x = torch.randn(16, 3, 224, 224, generator=torch.Generator().manual_seed(4)).to(DEV)
        _NETS[name] = test_block_eval_mb_gpu._network(name, x) if name.startswith("atomnas") else \
            test_fused_class_eval_gpu._network(name, 4, x).to(DEV).eval()
    return _NETS[name]


@pytest.fixture
def small_all(monkeypatch):
    from yet_another_mobilenet_series_b200 import engine
    monkeypatch.setattr(engine, "SMALL_BATCH_RULE", False)
    return engine


@pytest.mark.parametrize("name", ["atomnas_c", "atomnas_c+"])
def test_every_block_against_fp32(built_lib, small_all, name):
    """Every multi-branch block at N = 1 with the switch on: the split where eval_cluster_size
    picks it, against fp32 truth with the autocast yardstick; a second call gives the same bits."""
    from oracle import torch_model as tm
    engine = small_all
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model = _net(name)
    x = torch.randn(1, 3, 224, 224, generator=torch.Generator().manual_seed(3)).cuda()
    inputs = {}
    hooks = [b.register_forward_pre_hook(lambda mod, inp: inputs.__setitem__(id(mod), inp[0]))
             for b in multi_branch_blocks(model)]
    with torch.no_grad():
        model(x)
    for h in hooks:
        h.remove()
    split = 0
    for i, blk in enumerate(multi_branch_blocks(model)):
        xin = inputs[id(blk)].float()
        c0, s0 = engine.EVAL_MB_CALLS, engine.EVAL_MB_CLUSTER_CALLS
        engine.EVAL_SMALL_BATCH = True
        try:
            with torch.no_grad():
                y = blk(xin).float()
                y2 = blk(xin).float()
        finally:
            engine.EVAL_SMALL_BATCH = False
        torch.cuda.synchronize()
        assert engine.EVAL_MB_CALLS - c0 == 2
        split += engine.EVAL_MB_CLUSTER_CALLS - s0
        assert torch.equal(y, y2)
        ref = tm.as_reference(copy.deepcopy(blk)).eval()
        with torch.no_grad():
            yt = ref(xin)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                ya = ref(xin.contiguous(memory_format=torch.channels_last)).float()
        eo, ea = _rel(y, yt), _rel(ya, yt)
        print("%s block %d %s: vs fp32 %.3e autocast %.3e" % (name, i, engine.mb_kind(blk), eo, ea))
        assert eo <= SLACK * ea + FLOOR, (i, eo, ea)
    assert split > 0


def _evalstep(model, n, x, t, **kw):
    from yet_another_mobilenet_series_b200.trainer import EvalStep
    es = EvalStep(copy.deepcopy(model), n, use_graph=True, **kw)
    outs = []
    for _ in range(3):                  # eager warm-up, capture, replay
        es.evaluate([(x, t)])
        outs.append(es.logits.float().clone())
    assert es.phases["eval"].graph is not None
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2])
    return outs[-1]


@pytest.mark.parametrize("name", ["atomnas_c", "atomnas_c+", "autonl_l"])
@pytest.mark.parametrize("batch", [1, 2, 8])
def test_eval_step_network(built_lib, monkeypatch, name, batch):
    """EvalStep(small_batch=True), every covered kind on the path (rule off) and with the table as
    it stands, against fp32 truth with the autocast yardstick and against the default EvalStep;
    graph replay equals eager bitwise."""
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200 import engine
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model = _net(name)
    x = torch.randn(batch, 3, 224, 224, generator=torch.Generator().manual_seed(3)).bfloat16()
    t = torch.zeros(batch, dtype=torch.long)
    y_def = _evalstep(model, batch, x, t)
    c0 = engine.EVAL_MB_CALLS + engine.EVAL_FUSED_CALLS
    monkeypatch.setattr(engine, "SMALL_BATCH_RULE", False)
    y_all = _evalstep(model, batch, x, t, small_batch=True)
    assert engine.EVAL_MB_CALLS + engine.EVAL_FUSED_CALLS > c0
    monkeypatch.setattr(engine, "SMALL_BATCH_RULE", True)
    y_tab = _evalstep(model, batch, x, t, small_batch=True)
    ref = tm.as_reference(copy.deepcopy(model)).eval()
    with torch.no_grad():
        xr = x.float().to(DEV)
        yt = ref(xr).float()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ya = ref(xr.contiguous(memory_format=torch.channels_last)).float()
    ea = _rel(ya, yt)
    for tag, y in (("all kinds", y_all), ("table", y_tab)):
        eo, ed = _rel(y, yt), _rel(y, y_def)
        print("%s N=%d %s: vs fp32 %.3e autocast %.3e | vs default %.3e" % (name, batch, tag, eo, ea, ed))
        assert eo <= SLACK * ea + FLOOR, (tag, eo, ea)
        assert ed <= SLACK * ea + FLOOR, (tag, ed, ea)


@pytest.mark.parametrize("name", ["atomnas_c+", "autonl_l"])
def test_default_eval_step_unchanged(built_lib, monkeypatch, name):
    """Without small_batch the switch, the rule and the table change nothing: the same launches per
    forward and the same logits bit for bit, with every kind listed."""
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    model = _net(name)
    x = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(3)).bfloat16()
    t = torch.zeros(2, dtype=torch.long)

    def run():
        l0, m0, f0 = engine.LAUNCHES, engine.EVAL_MB_CALLS, engine.EVAL_FUSED_CALLS
        y = _evalstep(model, 2, x, t)
        return y, engine.LAUNCHES - l0, engine.EVAL_MB_CALLS - m0, engine.EVAL_FUSED_CALLS - f0

    y0, l0, m0, f0 = run()
    kinds = {engine.small_batch_kind(b) for b in model.modules()
             if isinstance(b, (mb.InvertedResidualChannels, mb.InvertedResidualChannelsFused))}
    monkeypatch.setattr(engine, "SMALL_BATCH_FASTER", tuple((k, 1 << 20) for k in kinds))
    y1, l1, m1, f1 = run()
    monkeypatch.setattr(engine, "SMALL_BATCH_RULE", False)
    y2, l2, m2, f2 = run()
    assert torch.equal(y0, y1) and torch.equal(y0, y2)
    assert l0 == l1 == l2 and m0 == m1 == m2 == 0 and f0 == f1 == f2
    assert engine.EVAL_SMALL_BATCH is False
