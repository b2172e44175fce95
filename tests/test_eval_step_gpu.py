"""GPU: validation on the sm_90a path (reference train.py:273-309): TrainStep.ema_model,
EvalStep.calibrate / evaluate and TrainStep.validate, on MobileNetV2, AutoNL-L (SE, non-local,
fused-class eval path) and AtomNAS-C+ (multi-branch four-launch fallback, padded shadow blocks).

- graph replays compute the eager bits (logits, sums, running statistics, num_batches_tracked),
  including a partial last batch, which runs eagerly in both;
- two calibrations from the same state give the same bits;
- EMA-model logits and calibrated statistics against the reference's stock-torch graph in fp32
  (DESIGN §c gate 2: err(ours) <= 1.5 err(autocast) + 2.5e-3), and the result keys against those
  of the fp32 logits (top-1 / top-5 flips reported);
- the EMA model holds the optimizer's shadows, never reads the live bf16 mirror, and is refreshed
  in place under a captured graph;
- validating between training steps leaves the training bits unchanged."""
import copy
import gc

import pytest
import torch

from _cfg import build_from_cfg

pytestmark = pytest.mark.gpu
CONFIGS = ["mobilenet_v2", "autonl_l", "atomnas_c+"]
B, SIZE, CLASSES = 8, 224, 100
SLACK, FLOOR = 1.5, 2.5e-3


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _batches(seed, sizes):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(n, 3, SIZE, SIZE, generator=g).bfloat16(),
             torch.randint(0, CLASSES, (n,), generator=g)) for n in sizes]


def _model(name, seed=5):
    model, _ = build_from_cfg(name, seed=seed, num_classes=CLASSES)
    return model.cuda()


def _trained(name, steps=2):
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    model = _model(name)
    ts = TrainStep(model, B, image_size=SIZE)
    for x, t in _batches(1, [B] * steps):
        ts(x, t)
    torch.cuda.synchronize()
    return ts


def _stats(model):
    return {k: v.clone() for k, v in model.named_buffers()
            if "running_" in k or "num_batches_tracked" in k}


def _same(a, b):
    return [k for k in a if not torch.equal(a[k], b[k])]


@pytest.mark.parametrize("name", CONFIGS)
def test_graph_equals_eager_and_determinism(built_lib, name):
    from yet_another_mobilenet_series_b200.trainer import EvalStep
    base = _model(name).eval()
    calib = _batches(2, [B, B, B])
    val = _batches(3, [B, B, 3])                     # two full batches and a partial one
    runs = {}
    for tag, graph in (("eager", False), ("graph", True), ("graph2", True)):
        m = copy.deepcopy(base)
        es = EvalStep(m, B, image_size=SIZE, use_graph=graph)
        es.calibrate(calib, steps=3)
        st = _stats(m)
        res = es.evaluate(val)
        runs[tag] = (st, res, es.loss_sum.clone(), es.counts.clone(), es.logits.clone())
        if graph:
            assert es.phases["calib"].graph is not None and es.phases["eval"].graph is not None
        del es, m
        gc.collect()
    e, g, g2 = runs["eager"], runs["graph"], runs["graph2"]
    assert all(int(v) == 3 for k, v in e[0].items() if "num_batches_tracked" in k)
    assert not _same(e[0], g[0]), _same(e[0], g[0])[:5]
    assert not _same(g[0], g2[0]), _same(g[0], g2[0])[:5]     # two calibrations, same bits
    for i in (2, 3, 4):
        assert torch.equal(e[i], g[i]) and torch.equal(g[i], g2[i]), i
    assert e[1] == g[1] == g2[1]
    assert int(e[3][2]) == 2 * B + 3
    # the same images evaluated eagerly, batch by batch, with the calibrated statistics: the
    # per-batch sums add up to the graph run's (partial last batch included)
    m = copy.deepcopy(base)
    with torch.no_grad():
        for k, v in m.named_buffers():
            if k in e[0]:
                v.copy_(e[0][k])
    es = EvalStep(m, B, image_size=SIZE, use_graph=False)
    loss_sum, counts = 0.0, torch.zeros_like(e[3])
    for batch in val:
        es.evaluate([batch])
        loss_sum += float(es.loss_sum)
        counts += es.counts
    assert torch.equal(counts, g[3])
    assert abs(loss_sum - float(g[2])) <= 1e-12 * abs(float(g[2]))


@pytest.mark.parametrize("name", CONFIGS)
def test_ema_model_and_reference_parity(built_lib, name):
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200.trainer import EvalStep
    rows = []
    ts = _trained(name)
    ema = ts.ema_model()
    # the EMA model holds the optimizer's shadows, bit for bit, and never the live mirror
    for q, p in zip(ema.parameters(), ts.model.parameters()):
        assert torch.equal(q, ts.opt.ema_shadow(p))
        assert getattr(q, "_yamb_bf16", None) is None and q.grad is None
    ema_stats = [b for n, b in ema.named_buffers() if "running_mean" in n or "running_var" in n]
    assert all(torch.equal(a, b) for a, b in zip(ema_stats, ts.stat_shadow))
    x = _batches(4, [B])[0][0].cuda()
    with torch.no_grad():
        ema.eval()
        ts.model.eval()
        y_ema, y_live = ema(x), ts.model(x)
        ts.model.train()
    assert not torch.equal(y_ema, y_live)
    # parity with the reference's stock-torch graph in fp32: calibration, then evaluation
    calib = _batches(5, [B, B])
    val = _batches(6, [B, B])
    ref = tm.as_reference(copy.deepcopy(ema)).cuda()
    ref_a = tm.as_reference(copy.deepcopy(ema)).cuda().to(memory_format=torch.channels_last)

    def bn_calibration(m):                           # reference utils/common.py:175-187
        if isinstance(m, torch.nn.BatchNorm2d):
            m.reset_running_stats()
            m.train()
            m.momentum = None

    es = EvalStep(ema, B, image_size=SIZE)
    es.calibrate(calib)
    for r in (ref, ref_a):
        r.eval()
        r.apply(bn_calibration)
    with torch.no_grad():
        for xc, _ in calib:
            ref(xc.float().cuda())
            with torch.autocast("cuda", dtype=torch.bfloat16):
                ref_a(xc.float().cuda().contiguous(memory_format=torch.channels_last))
    bo, bt, ba = (dict(m.named_buffers()) for m in (ema, ref, ref_a))
    ks = [k for k in bt if "running_" in k]
    mo = sum(_rel(bo[k], bt[k]) for k in ks) / len(ks)
    ma = sum(_rel(ba[k], bt[k]) for k in ks) / len(ks)
    rows.append("%s calibrated statistics: ours %.2e autocast %.2e" % (name, mo, ma))
    assert mo <= SLACK * ma + FLOOR, rows
    assert all(int(bo[k]) == int(bt[k]) == 2 for k in bt if k.endswith("num_batches_tracked"))
    res = es.evaluate(val)
    ref.eval()
    ref_a.eval()
    lt, la, lo = [], [], []
    with torch.no_grad():
        for xv, tv in val:
            lt.append(ref(xv.float().cuda()))
            with torch.autocast("cuda", dtype=torch.bfloat16):
                la.append(ref_a(xv.float().cuda().contiguous(memory_format=torch.channels_last)).float())
            es_single = es.logits                    # logits of the batch just evaluated last
        lt, la = torch.cat(lt), torch.cat(la)
        with torch.no_grad():
            ema.eval()
            from yet_another_mobilenet_series_b200 import engine
            engine.EVAL_TAIL_FUSED = True
            try:
                lo = torch.cat([ema(xv.cuda()) for xv, _ in val])
            finally:
                engine.EVAL_TAIL_FUSED = False
    assert torch.equal(lo[-B:], es_single)           # the graph's logits are the eager ones
    eo, ea = _rel(lo, lt), _rel(la, lt)
    rows.append("%s EMA-model logits: ours %.2e autocast %.2e" % (name, eo, ea))
    assert eo <= SLACK * ea + FLOOR, rows
    tt = torch.cat([tv for _, tv in val]).cuda()
    n = tt.numel()
    top5 = lt.topk(5, 1).indices
    ref_res = {"loss": float(torch.nn.functional.cross_entropy(lt, tt)),
               "top1_error": 1.0 - float((top5[:, 0] == tt).double().mean()),
               "top5_error": 1.0 - float((top5 == tt[:, None]).any(1).double().mean())}
    o5 = lo.topk(5, 1).indices
    flips1 = int(((o5[:, 0] == tt) != (top5[:, 0] == tt)).sum())
    flips5 = int(((o5 == tt[:, None]).any(1) != (top5 == tt[:, None]).any(1)).sum())
    rows.append("%s results ours %s reference(fp32 logits) %s flips top1 %d top5 %d of %d"
                % (name, res, ref_res, flips1, flips5, n))
    print("\n".join(rows))
    assert abs(res["top1_error"] - ref_res["top1_error"]) * n <= flips1
    assert abs(res["top5_error"] - ref_res["top5_error"]) * n <= flips5
    assert abs(res["loss"] - ref_res["loss"]) <= 2 * SLACK * ea * max(1.0, ref_res["loss"]) + FLOOR
    # a second ema_model() after more steps: the same copy, refreshed in place, seen by the graph
    addrs = [p.data_ptr() for p in ema.parameters()]
    for xb, tb in _batches(7, [B, B]):
        ts(xb, tb)
    ema2 = ts.ema_model()
    assert ema2 is ema and [p.data_ptr() for p in ema2.parameters()] == addrs
    for q, p in zip(ema2.parameters(), ts.model.parameters()):
        assert torch.equal(q, ts.opt.ema_shadow(p))
    g_before = es.phases["eval"].graph
    res2 = es.evaluate(val)
    assert es.phases["eval"].graph is g_before       # replayed, not re-captured
    fresh = EvalStep(copy.deepcopy(ema2), B, image_size=SIZE, use_graph=False)
    assert fresh.evaluate(val) == res2
    assert res2 != res


@pytest.mark.parametrize("name", ["mobilenet_v2", "autonl_l"])
def test_validation_does_not_perturb_training(built_lib, name):
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    k = 3
    train = _batches(8, [B] * (2 * k))
    calib = _batches(9, [B, B])
    val = _batches(10, [B, B, 5])
    out = []
    for validate in (True, False):
        model = _model(name)
        ts = TrainStep(model, B, image_size=SIZE)
        for i, (x, t) in enumerate(train):
            if validate and i == k:
                res = ts.validate(val, calib_batches=calib, calib_steps=2)
                assert set(res) == {"loss", "top1_error", "top5_error"}
            ts(x, t)
        torch.cuda.synchronize()
        A = ts.opt.arenas()
        snap = {a: A[a].clone() for a in ("p", "sq", "mom", "ema", "bf16") if A.get(a) is not None}
        snap.update({"buf." + n: b.clone() for n, b in model.named_buffers()})
        snap.update({"shadow.%d" % i: s.clone() for i, s in enumerate(ts.stat_shadow)})
        out.append(snap)
        del ts, model
        gc.collect()
    assert not _same(out[0], out[1]), _same(out[0], out[1])[:5]
