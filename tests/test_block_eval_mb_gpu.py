"""Multi-branch eval path (csrc/block_eval_mb.cu, engine.eval_forward_mb) on the GPU:
  * every compiled instantiation (tile geometry x lean / generic activation x plain / gate / pool)
    through the C ABI, element by element against the fp64 intervals of tests/block_eval_ref64.py
    applied per 64-channel slice with the slice's own kernel, on packed blocks whose group
    boundaries fall inside slices (multi-tile walks, odd image counts, stride 2 down to one pixel);
  * the packing kernel against a gather of the module's tensors, bit for bit;
  * every multi-branch block of AtomNAS-C and C+ against fp32 truth with the autocast yardstick;
  * whole-network eval logits of the six AtomNAS configs, the flag off leaving the default path;
  * EvalStep(fused_multi_branch=True): graph replay equals eager bitwise, reruns give the same bits,
    calibration then evaluation end to end."""
import copy
import ctypes as C

import pytest
import torch

import block_eval_ref64 as br
from test_block_eval_mb_cpu import build, multi_branch_blocks

pytestmark = pytest.mark.gpu
DEV = "cuda"
SLACK, FLOOR = 1.5, 2.5e-3


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ---- kernel instantiations against fp64 ------------------------------------------------------------
# (kmax, stride, N, H, Cin, Cout, groups [(k, channels)]): one case per tile geometry of
# block_eval_mb_launch
GROUPS7 = [(7, 72), (5, 64), (3, 64)]     # slices: k7 | k7 (7|5 at 72) | k5 (5|3 at 136) | k3
GROUPS5 = [(5, 72), (3, 64)]              # slices: k5 | k5 (5|3 at 72) | k3
CASES = [
    (5, 2, 3, 14, 40, 48, GROUPS5),       # EvGeomMB<5, 2, 6, 7, 1, 2>
    (5, 2, 2, 2, 32, 40, GROUPS5),        # stride 2 down to one output pixel
    (5, 1, 2, 28, 40, 40, GROUPS5),       # <5, 1, 7, 16, 1, 4>, multi-tile, residual
    (5, 1, 3, 7, 32, 40, GROUPS5),        # <5, 1, 7, 7, 2, 4>, odd image count
    (5, 1, 1, 14, 48, 192, GROUPS5),      # <5, 1, 7, 7, 1, 4>, wide project
    (7, 1, 2, 14, 80, 80, GROUPS7),       # <7, 1, 7, 7, 1, 2>, residual
    (7, 2, 3, 14, 40, 56, GROUPS7),       # <7, 2, 4, 7, 1, 2>
    (7, 2, 1, 2, 40, 56, GROUPS7),        # stride 2 down to one output pixel
]


def _case_tensors(case, act, seed):
    K, S, N, H, Cin, Cout, groups = case
    g = torch.Generator(device=DEV).manual_seed(seed)
    Chid = sum(c for _, c in groups)
    u = lambda *s, lo=0.0, hi=1.0: torch.rand(*s, generator=g, device=DEV) * (hi - lo) + lo
    x = (torch.randn(N, H, H, Cin, generator=g, device=DEV)).to(torch.bfloat16)
    w1 = (torch.randn(Chid, Cin, generator=g, device=DEV) / Cin ** 0.5).to(torch.bfloat16)
    w3 = (torch.randn(Cout, Chid, generator=g, device=DEV) / Chid ** 0.5).to(torch.bfloat16)
    taps = torch.zeros(Chid, K, K, device=DEV)
    c0 = 0
    for k, c in groups:
        o = (K - k) // 2
        taps[c0:c0 + c, o:o + k, o:o + k] = torch.randn(c, k, k, generator=g, device=DEV) / k
        c0 += c

    def bn(C):
        return {"gamma": u(C, lo=0.5, hi=1.5), "beta": torch.randn(C, generator=g, device=DEV) * 0.3,
                "mean": torch.randn(C, generator=g, device=DEV) * 0.3, "var": u(C, lo=0.5, hi=2.0),
                "eps": 1e-3}
    gate = u(N, Chid, lo=0.05, hi=1.0)
    return dict(x=x, w1=w1, w3=w3, taps=taps.contiguous(), bn1=bn(Chid), bn2=bn(Chid), bn3=bn(Cout),
                gate=gate, Chid=Chid)


def _args(case, t, act, mode, residual):
    from yet_another_mobilenet_series_b200 import native as nat
    K, S, N, H, Cin, Cout, groups = case
    m = nat.BlockEvalMb()
    a = m.base
    a.N, a.H, a.W, a.Cin, a.Chid, a.Cout = N, H, H, Cin, t["Chid"], Cout
    a.kernel, a.stride, a.act, a.residual = K, S, act, 1 if residual else 0
    a.x, a.w_expand, a.w_dw, a.w_project = (t["x"].data_ptr(), t["w1"].data_ptr(),
                                            t["taps"].data_ptr(), t["w3"].data_ptr())
    for dst, bn in ((a.bn1, t["bn1"]), (a.bn2, t["bn2"]), (a.bn3, t["bn3"])):
        dst.gamma, dst.beta = bn["gamma"].data_ptr(), bn["beta"].data_ptr()
        dst.running_mean, dst.running_var, dst.eps = bn["mean"].data_ptr(), bn["var"].data_ptr(), bn["eps"]
    m.ngroups = len(groups)
    c0 = 0
    for i, (k, c) in enumerate(groups):
        m.group_k[i], m.group_c0[i] = k, c0
        c0 += c
    if mode == "gate":
        a.gate = t["gate"].data_ptr()
    return m


def _reference(case, t, act, mode, residual):
    """fp64 intervals: expand over every hidden channel, the stencil per 64-channel slice with the
    kernel of its first channel over the centred window of the zero-embedded taps."""
    K, S, N, H, Cin, Cout, groups = case
    x = t["x"].permute(0, 3, 1, 2).double()
    a_lo, a_hi = br.expand(x, t["w1"], t["bn1"], act)
    bounds = [sum(c for _, c in groups[:i]) for i in range(len(groups))]
    los, his = [], []
    for s0 in range(0, t["Chid"], 64):
        kc = [k for (k, _), b0 in zip(groups, bounds) if b0 <= s0][-1]
        o = (K - kc) // 2
        sl = slice(s0, min(s0 + 64, t["Chid"]))
        w = t["taps"][sl, o:o + kc, o:o + kc].reshape(-1, kc * kc)
        bn2 = {k: (v[sl] if torch.is_tensor(v) else v) for k, v in t["bn2"].items()}
        lo, hi = br.stencil(a_lo[:, sl], a_hi[:, sl], w, kc, S, bn2, act)
        los.append(lo)
        his.append(hi)
    lo, hi = torch.cat(los, 1), torch.cat(his, 1)
    if mode == "pool":
        return br.pooled(lo, hi, 64)
    if mode == "gate":
        lo, hi = br.gated(lo, hi, t["gate"])
    return br.project(lo, hi, t["w3"], t["bn3"], x if residual else None)


@pytest.mark.parametrize("case", CASES, ids=lambda c: "k%d_s%d_n%d_h%d_co%d" % (c[:4] + (c[5],)))
@pytest.mark.parametrize("act", [1, 3], ids=["relu", "swish"])
def test_instantiations_against_fp64(built_lib, case, act):
    from yet_another_mobilenet_series_b200 import native as nat
    K, S, N, H, Cin, Cout, groups = case
    Ho = (H - 1) // S + 1
    for mode, seed in (("plain", 1), ("gate", 2), ("pool", 3)):
        t = _case_tensors(case, act, seed + 10 * act)
        residual = mode == "plain" and S == 1 and Cin == Cout
        m = _args(case, t, act, mode, residual)
        if mode == "pool":
            out = torch.full((N * t["Chid"] + 8,), 7.0, device=DEV)
            m.base.pooled = out.data_ptr()
            nat.check(built_lib.yamb_block_eval_mb_pool_fwd(C.byref(m), nat.stream_handle()))
            got = out[:-8].view(N, t["Chid"]).double()
        else:
            out = torch.full((N * Ho * Ho * Cout + 8,), 7.0, device=DEV, dtype=torch.bfloat16)
            m.base.y = out.data_ptr()
            nat.check(built_lib.yamb_block_eval_mb_fwd(C.byref(m), nat.stream_handle()))
            got = out[:-8].view(N, Ho, Ho, Cout).permute(0, 3, 1, 2).double()
        torch.cuda.synchronize()
        assert (out[-8:].float() == 7.0).all(), "guard values overwritten"
        lo, hi = _reference(case, t, act, mode, residual)
        bad = ~((got >= lo) & (got <= hi))
        assert not bad.any(), (mode, int(bad.sum()), got[bad][:4], lo[bad][:4], hi[bad][:4])


def test_pack_kernel_bitwise(built_lib):
    """yamb_block_eval_mb_pack writes the gather of the module's tensors (bf16 round to nearest of
    the 1x1 weights), zero-embedded taps and the padding BatchNorms, SE included."""
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    torch.manual_seed(0)
    for cls, kw in ((mb.InvertedResidualChannelsFused, {"se_ratio": 0.25}),
                    (mb.InvertedResidualChannels, {})):
        block = cls(24, 32, 1, [37, 61, 70], [3, 5, 7], True, active_fn=mb.get_active_fn("nn.Swish"),
                    batch_norm_kwargs={"momentum": 0.01, "eps": 1e-3}, **kw).cuda().eval()
        for m in block.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.data.uniform_(0.5, 1.5)
                m.bias.data.normal_(0, 0.3)
                m.running_mean.normal_(0, 0.5)
                m.running_var.uniform_(0.5, 2.0)
        parts = engine.block_parts(block)
        R = parts.se.se_reduce.weight.shape[0] if parts.se is not None else 0
        ms = engine._mb_state(block, torch.device(DEV), R)
        engine.launch(built_lib.yamb_block_eval_mb_pack, engine._mb_pack_args(block, parts, ms))
        torch.cuda.synchronize()
        lay = ms["layout"]
        code = torch.tensor(lay.map)
        offs = [0, 37, 98]
        for b, k in enumerate(block.kernel_sizes):
            js = torch.nonzero((code >= 0) & ((code >> 16) == b)).flatten().to(DEV)
            c = (code[code >= 0][(code[code >= 0] >> 16) == b] & 0xFFFF).to(DEV)
            if parts.fused:
                src, w1, w3, bn1 = offs[b] + c, parts.expand_convs[0].weight, parts.project_convs[0].weight, parts.bn1s[0]
            else:
                src, w1, w3, bn1 = c, parts.expand_convs[b].weight, parts.project_convs[b].weight, parts.bn1s[b]
            assert torch.equal(ms["w1"][js], w1[src, :, 0, 0].to(torch.bfloat16))
            assert torch.equal(ms["w3"][:, js], w3[:, src, 0, 0].to(torch.bfloat16))
            o = (7 - k) // 2
            want = torch.zeros(len(js), 7, 7, device=DEV)
            want[:, o:o + k, o:o + k] = parts.dws[b][0].weight[c, 0]
            assert torch.equal(ms["wdw"][js], want)
            bn2 = parts.dws[b][1]
            assert torch.equal(ms["bn1"][:, js], torch.stack([bn1.weight[src], bn1.bias[src],
                                                              bn1.running_mean[src], bn1.running_var[src]]))
            assert torch.equal(ms["bn2"][:, js], torch.stack([bn2.weight[c], bn2.bias[c],
                                                              bn2.running_mean[c], bn2.running_var[c]]))
            if parts.se is not None:
                se = parts.se
                assert torch.equal(ms["se"][0][:, js], se.se_reduce.weight[:, offs[b] + c, 0, 0])
                assert torch.equal(ms["se"][1][js], se.se_expand.weight[offs[b] + c, :, 0, 0])
                assert torch.equal(ms["se"][2][js], se.se_expand.bias[offs[b] + c])
        pad = (code < 0).to(DEV)
        assert (ms["w1"][pad] == 0).all() and (ms["w3"][:, pad] == 0).all() and (ms["wdw"][pad] == 0).all()
        want_pad = torch.tensor([0.0, 0.0, 0.0, 1.0], device=DEV)[:, None]
        assert torch.equal(ms["bn1"][:, pad], want_pad.expand(4, int(pad.sum())))
        assert torch.equal(ms["bn2"][:, pad], want_pad.expand(4, int(pad.sum())))


# ---- modules and networks ----------------------------------------------------------------------
def _network(name, x):
    """Model of the config with SE biases and BatchNorm running statistics calibrated on x by the
    stock-torch graph."""
    from oracle import torch_model as tm
    model = build(name)
    g = torch.Generator().manual_seed(5)
    for m in model.modules():
        if isinstance(m, torch.nn.Conv2d) and m.bias is not None:
            m.bias.data.normal_(0, 0.3, generator=g)
    ref = tm.as_reference(model).cuda().train()
    for m in ref.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.reset_running_stats()
            m.momentum = None
    with torch.no_grad():
        ref(x)
    model.load_state_dict({k: v.cpu() for k, v in ref.state_dict().items()})
    return model.cuda().eval()


@pytest.fixture
def mb_on(monkeypatch):
    from yet_another_mobilenet_series_b200 import engine
    monkeypatch.setattr(engine, "EVAL_MULTI_BRANCH", True)
    monkeypatch.setattr(engine, "MB_SHAPE_RULE", False)
    return engine


@pytest.mark.parametrize("name", ["atomnas_c", "atomnas_c+"])
def test_every_block_against_fp32(built_lib, mb_on, name):
    """Every multi-branch block at its 224x224-derived input size, one call each (pack + kernel,
    + pool pass and gate FCs with SE), against fp32 truth with the autocast yardstick."""
    from oracle import torch_model as tm
    engine = mb_on
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    x = torch.randn(4, 3, 224, 224, generator=torch.Generator().manual_seed(3)).cuda()
    model = _network(name, x)
    inputs = {}
    hooks = [b.register_forward_pre_hook(lambda mod, inp: inputs.__setitem__(id(mod), inp[0]))
             for b in multi_branch_blocks(model)]
    with torch.no_grad():
        engine.EVAL_MULTI_BRANCH = False
        model(x)
        engine.EVAL_MULTI_BRANCH = True
    for h in hooks:
        h.remove()
    for i, blk in enumerate(multi_branch_blocks(model)):
        xin = inputs[id(blk)].float()
        c0, l0 = engine.EVAL_MB_CALLS, engine.LAUNCHES
        with torch.no_grad():
            y = blk(xin).float()
            y2 = blk(xin).float()
        torch.cuda.synchronize()
        assert engine.EVAL_MB_CALLS - c0 == 2
        assert engine.LAUNCHES - l0 == 2 * (4 if engine.block_parts(blk).se is not None else 2)
        assert torch.equal(y, y2)
        ref = tm.as_reference(copy.deepcopy(blk)).eval()
        with torch.no_grad():
            yt = ref(xin)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                ya = ref(xin.contiguous(memory_format=torch.channels_last)).float()
        eo, ea = _rel(y, yt), _rel(ya, yt)
        print("%s block %d %s: vs fp32 %.3e autocast %.3e" % (name, i, engine.mb_kind(blk), eo, ea))
        assert eo <= SLACK * ea + FLOOR, (i, eo, ea)


@pytest.mark.parametrize("name", ["atomnas_a", "atomnas_b", "atomnas_c", "atomnas_a+", "atomnas_b+",
                                  "atomnas_c+"])
def test_network_logits(built_lib, mb_on, name):
    """Whole network in eval() under no_grad with the flag on: every multi-branch block on the path,
    logits against the stock-torch graph in fp32 with the autocast yardstick and against the
    default path; with the flag off no block takes it."""
    from oracle import torch_model as tm
    engine = mb_on
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    x = torch.randn(8, 3, 224, 224, generator=torch.Generator().manual_seed(3)).cuda()
    model = _network(name, x)
    nmb = len(multi_branch_blocks(model))
    c0 = engine.EVAL_MB_CALLS
    with torch.no_grad():
        y = model(x).float()
    torch.cuda.synchronize()
    assert engine.EVAL_MB_CALLS - c0 == nmb
    engine.EVAL_MULTI_BRANCH = False
    with torch.no_grad():
        y_off = model(x).float()
    assert engine.EVAL_MB_CALLS - c0 == nmb
    ref = tm.as_reference(copy.deepcopy(model)).eval()
    with torch.no_grad():
        yt = ref(x)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ya = ref(x.contiguous(memory_format=torch.channels_last)).float()
    eo, ea, ed = _rel(y, yt), _rel(ya, yt), _rel(y, y_off)
    print("%s: vs fp32 %.3e autocast %.3e | vs default path %.3e" % (name, eo, ea, ed))
    assert eo <= SLACK * ea + FLOOR, (eo, ea)


def test_eval_step(built_lib, mb_on):
    """EvalStep(fused_multi_branch=True) on AtomNAS-C+: graph replay equals eager bitwise, a second
    run the same bits, calibration then evaluation end to end; the flag is off outside the step."""
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import EvalStep
    x = torch.randn(16, 3, 224, 224, generator=torch.Generator().manual_seed(3))
    model = _network("atomnas_c+", x.cuda())
    t = torch.randint(0, 1000, (16,), generator=torch.Generator().manual_seed(4))
    batches = [(x[:8], t[:8]), (x[8:], t[8:])]
    logits = {}
    for use_graph in (False, True):
        es = EvalStep(model, 8, use_graph=use_graph, fused_multi_branch=True)
        c0 = engine.EVAL_MB_CALLS
        outs = []
        for _ in range(3):                  # warm-up, capture, replay
            es.evaluate(batches[:1])
            outs.append(es.logits.clone())
        torch.cuda.synchronize()
        assert engine.EVAL_MB_CALLS > c0
        assert torch.equal(outs[1], outs[2]) and torch.equal(outs[0], outs[1])
        logits[use_graph] = outs[-1]
    assert torch.equal(logits[False], logits[True])
    es = EvalStep(model, 8, fused_multi_branch=True)
    es.calibrate(batches, 2)
    res = es.evaluate(batches)
    assert res["loss"] == res["loss"] and 0.0 <= res["top1_error"] <= 1.0
