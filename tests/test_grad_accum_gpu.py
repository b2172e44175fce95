"""GPU: TrainStep with gradient accumulation (`micro_batch`).

1. micro_batch=None and micro_batch=per_gpu_batch are the same step, bit for bit.
2. per_gpu_batch 16 in micro-batches of 4 against the reference step sequence running the same
   micro-batches (the mean loss of each pass weighted by n_i / n, one L2 term, one optimizer step,
   one EMA update per step) in fp32 (truth) and under autocast-bf16 (yardstick), with the rule of
   tests/test_configs_gpu.py: err(ours) <= 2 err(autocast) + 5e-3 on the loss (relative, mean over
   the steps), err(ours) <= 1.5 err(autocast) + 2.5e-3 on the >= 2-D weights (their updates and
   EMA shadows, error per tensor, mean and 90th percentile over the tensors), on the 1-D parameters together and on the
   running statistics and their EMA shadows (per buffer, mean and 90th percentile).  Per-tensor
   and per-step errors are aggregated because BatchNorm over micro-batches of 4 images makes a
   single tensor's three-step trajectory noise-dominated for the autocast yardstick as well (at
   64 x 64, MobileNetV2's updates differ from the fp32 ones by more than their own norm, for both).
   MobileNetV2 and AtomNAS-C+ (multi-branch, SE, Swish, padded widths) with RMSprop, MobileNetV2
   with Nesterov SGD and the 'slimmable' L2, and a partial last batch of 10 (micro-batches 4, 4,
   2) between full ones, after which the captured graph replays the next full batch.
3. The k = 4 step as a CUDA-graph replay equals the eager step bit for bit; two fresh runs give
   the same bits; save_status after step 2 and a resumed step 3 equal the uninterrupted run, and
   the checkpoint loads into a TrainStep without micro-batches.
Dropout is off: its stream differs between capture and eager, and between us and the reference."""
import importlib
import sys
import types

import pytest
import torch

from _cfg import MODULE_MAP, load_cfgs
from test_checkpoint_gpu import _same, _snap
from test_configs_gpu import _rel
from test_model_gpu import _restore, _state

pytestmark = pytest.mark.gpu
B, MICRO = 16, 4
SIZE = {"mbv2": 128, "atomnas_c+": 128}
OPT = {"rmsprop": {}, "sgd": dict(optimizer="sgd", nesterov=True,
                                  weight_decay_method="slimmable", base_lr=0.1)}


@pytest.fixture
def flags(monkeypatch):
    """A stand-in for the reference's utils.config (blocks of the searched networks read FLAGS)."""
    mod = types.ModuleType("utils.config")
    mod.FLAGS = types.SimpleNamespace()
    monkeypatch.setitem(sys.modules, "utils.config", mod)
    return mod


def _model(kind, seed=5):
    """CPU model: MobileNetV2 (the reference's yml) or AtomNAS-C+, 100 classes, dropout off."""
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    name = "mobilenet_v2" if kind == "mbv2" else kind
    cfg = load_cfgs()[name]
    lib = importlib.import_module(MODULE_MAP[cfg["flags"]["model"]])
    kw = dict(cfg["model_kwparams"])
    kw.update(num_classes=100, input_size=SIZE[kind])
    torch.manual_seed(seed)
    model = lib.Model(**kw)
    model.apply(mb.init_weights_mnas)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    return model


def _batch(kind, i, n=B):
    g = torch.Generator().manual_seed(200 + i)
    return (torch.randn(n, 3, SIZE[kind], SIZE[kind], generator=g).to(torch.bfloat16),
            torch.randint(0, 100, (n,), generator=g))


def _ts(kind, model, opt="rmsprop", micro=MICRO, **kw):
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    return TrainStep(model, B, image_size=SIZE[kind], micro_batch=micro, **OPT[opt], **kw)


# ---- the reference step sequence over micro-batches ---------------------------------------------
def _ref_step(tr, x, t, micro):
    """train.py:64-114 with the batch split into passes of `micro` rows: each backpropagates its
    mean loss x n_i / n; then the L2 term once, one optimizer step, one EMA update.  Returns the
    mean loss over the n rows (without L2)."""
    from oracle import torch_model as tm
    model = tr.model
    model.train()
    tr.opt.zero_grad()
    n, total = x.shape[0], 0.0
    for s in range(0, n, micro):
        xs, ts = x[s:s + micro], t[s:s + micro]
        if tr.autocast is not None:
            with torch.autocast("cuda", dtype=tr.autocast):
                out = model(xs).float()
        else:
            out = model(xs)
        lv = tm.label_smooth_ce(out, ts, tr.smoothing)
        (lv.mean() * (xs.shape[0] / n)).backward()
        total += float(lv.detach().double().sum())
    tr.l2_loss(model, tr.wd).backward()
    tr.opt.step()
    tr.global_step += 1
    named = dict(model.named_parameters())
    named.update(dict(model.named_buffers()))
    for k in tr.ema.shadow:
        tr.ema(k, named[k], tr.global_step)
    return total / n


def _flat(ts):
    return torch.cat([t.detach().double().flatten().cpu() for t in ts])


def _check(rows, what, eo, ea, factor=1.5, slack=2.5e-3):
    rows.append("%-48s ours %.3e autocast %.3e" % (what, eo, ea))
    return eo <= factor * ea + slack


def _vs_reference(kind, opt, sizes):
    import sgd_oracle as so
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda")
    model = _model(kind)
    ref_kw = dict(OPT[opt])
    ref32 = so.RefTrainer(so.tm.as_reference(model).to(dev), B, **ref_kw)
    ref16 = so.RefTrainer(so.tm.as_reference(model).to(dev).to(memory_format=torch.channels_last),
                          B, autocast=torch.bfloat16, **ref_kw)
    p0 = {k: v.detach().clone() for k, v in model.named_parameters()}
    model = model.to(dev)
    ts = _ts(kind, model, opt)
    rows, bad, graphs = ["%s %s sizes %s micro %d" % (kind, opt, sizes, MICRO)], [], []
    lerr = []
    for i, n in enumerate(sizes):
        x, t = _batch(kind, i, n)
        xd, td = x.to(dev).float(), t.to(dev)
        l32 = _ref_step(ref32, xd, td, MICRO)
        l16 = _ref_step(ref16, xd.contiguous(memory_format=torch.channels_last), td, MICRO)
        lo = float(ts(x, t))
        graphs.append(ts.graph)
        lerr.append((abs(lo - l32) / abs(l32), abs(l16 - l32) / abs(l32)))
        rows.append("loss step %d (n=%d): ours %.5f fp32 %.5f autocast %.5f" % (i, n, lo, l32, l16))
    if not _check(rows, "loss, mean relative error over the steps",
                  sum(e for e, _ in lerr) / len(lerr), sum(a for _, a in lerr) / len(lerr),
                  factor=2.0, slack=5e-3):
        bad.append("loss")
    torch.cuda.synchronize()
    po, pt, pa = (dict(m.named_parameters()) for m in (model, ref32.model, ref16.model))
    keys = list(po)
    big = [k for k in keys if po[k].dim() >= 2]
    small = [k for k in keys if po[k].dim() < 2]
    shadow = {k: ts.opt.ema_shadow(po[k]) for k in keys}
    p0d = {k: v.to(dev) for k, v in p0.items()}

    def upd(d, ks):
        return _flat([d[k] - p0d[k] for k in ks])

    for what, d32, d16, dour in (("update", pt, pa, po),
                                 ("ema", ref32.ema.shadow, ref16.ema.shadow, shadow)):
        eo = sorted(_rel(upd(dour, [k]), upd(d32, [k])) for k in big)
        ea = sorted(_rel(upd(d16, [k]), upd(d32, [k])) for k in big)
        i90 = int(0.9 * (len(eo) - 1))
        if not _check(rows, "%s of the >= 2-D weights, per-tensor mean" % what,
                      sum(eo) / len(eo), sum(ea) / len(ea)):
            bad.append("%s >= 2-D mean" % what)
        if not _check(rows, "%s of the >= 2-D weights, per-tensor p90" % what, eo[i90], ea[i90]):
            bad.append("%s >= 2-D p90" % what)
    for what, d32, d16, dour in (("update", pt, pa, po),
                                 ("ema", ref32.ema.shadow, ref16.ema.shadow, shadow)):
        if not _check(rows, "%s of the 1-D parameters" % what, _rel(upd(dour, small),
                      upd(d32, small)), _rel(upd(d16, small), upd(d32, small))):
            bad.append("%s 1-D" % what)
    bo, bt, ba = (dict(m.named_buffers()) for m in (model, ref32.model, ref16.model))
    snames = [n for n in bo if "running_mean" in n or "running_var" in n]
    sho = dict(zip(snames, ts.stat_shadow))
    for what, our, truth, auto in (("running", bo, bt, ba),
                                   ("stat shadow", sho, ref32.ema.shadow, ref16.ema.shadow)):
        for kind_ in ("running_mean", "running_var"):
            ks = [k for k in snames if k.endswith(kind_)]
            eo = sorted(_rel(_flat([our[k]]), _flat([truth[k]])) for k in ks)
            ea = sorted(_rel(_flat([auto[k]]), _flat([truth[k]])) for k in ks)
            i90 = int(0.9 * (len(eo) - 1))
            if not _check(rows, "%s %s per-buffer mean" % (what, kind_), sum(eo) / len(eo),
                          sum(ea) / len(ea)):
                bad.append("%s %s mean" % (what, kind_))
            if not _check(rows, "%s %s per-buffer p90" % (what, kind_), eo[i90], ea[i90]):
                bad.append("%s %s p90" % (what, kind_))
    nbt = [k for k in bt if k.endswith("num_batches_tracked")]
    passes = sum(-(-n // MICRO) for n in sizes)
    assert all(int(bo[k]) == int(bt[k]) == passes for k in nbt)
    print("\n".join(rows + ["FAILED: %s" % bad]))
    assert not bad, (bad, rows)
    return ts, graphs


@pytest.mark.parametrize("kind,opt", [("mbv2", "rmsprop"), ("atomnas_c+", "rmsprop"),
                                      ("mbv2", "sgd")])
def test_micro_batches_vs_reference_sequence(built_lib, flags, kind, opt):
    ts, graphs = _vs_reference(kind, opt, [B, B, B])
    assert graphs[2] is not None and ts.launches_per_step is not None


def test_partial_last_batch_vs_reference_sequence(built_lib, flags):
    ts, graphs = _vs_reference("mbv2", "rmsprop", [B, B, B, 10, B])
    assert graphs[2] is not None and graphs[2] is graphs[3] is graphs[4]


# ---- bits ---------------------------------------------------------------------------------------
def _run(kind, micro, steps, **kw):
    ts = _ts(kind, _model(kind).cuda(), micro=micro, **kw)
    return ts, [_snap(ts, ts(*_batch(kind, i))) for i in range(steps)]


def test_micro_batch_of_the_whole_batch_is_the_plain_step(built_lib):
    a, sa = _run("mbv2", None, 3)
    b, sb = _run("mbv2", B, 3)
    assert a.graph is not None and b.graph is not None
    assert a.launches_per_step == b.launches_per_step
    for x, y in zip(sa, sb):
        _same(x, y)


def test_graph_replay_equals_eager(built_lib):
    """The same k = 4 step (same state, same batch) eagerly and as a CUDA-graph replay."""
    kind = "mbv2"
    ts, _ = _run(kind, MICRO, 2)                       # two eager warm-up steps
    x, t = _batch(kind, 7)
    torch.cuda.synchronize()
    st = _state(ts, ts.model)
    ts.use_graph = False
    eager = _snap(ts, ts(x, t))
    _restore(ts, ts.model, st)
    ts.use_graph = True
    graph = _snap(ts, ts(x, t))                         # captures, then replays
    assert ts.graph is not None
    # _restore leaves the optimizer's host-side step counters advanced: compare the rest
    _same(*({k: v for k, v in s.items() if not k.endswith(".step")} for s in (eager, graph)))
    # the launches of one MICRO-image step per micro-batch, plus the optimizer kernel
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    one = TrainStep(_model(kind).cuda(), MICRO, image_size=SIZE[kind])
    one(x[:MICRO], t[:MICRO])
    assert ts.launches_per_step - 1 == (B // MICRO) * (one.launches_per_step - 1)


def test_two_fresh_runs_same_bits(built_lib):
    _, a = _run("mbv2", MICRO, 4)
    _, b = _run("mbv2", MICRO, 4)
    for x, y in zip(a, b):
        _same(x, y)


def test_resume_after_step_2(built_lib, tmp_path):
    kind = "mbv2"
    _, full = _run(kind, MICRO, 3)
    ts, part = _run(kind, MICRO, 2)
    path = str(tmp_path / "latest_checkpoint.pt")
    ts.save_status(path, 0, 0.5, None)
    ck = torch.load(path, map_location="cpu")
    del ts
    resumed = _ts(kind, _model(kind, seed=6).cuda())    # another init: all of it is loaded
    resumed.load_state_dict(ck)
    _same(full[2], _snap(resumed, resumed(*_batch(kind, 2))))
    # micro_batch is not checkpoint content: the same file continues without micro-batches
    plain = _ts(kind, _model(kind, seed=6).cuda(), micro=None)
    plain.load_state_dict(ck)
    after = _snap(plain, part[1]["loss"])
    _same(part[1], after)
    assert torch.isfinite(plain(*_batch(kind, 2))) and plain.global_step == 3
