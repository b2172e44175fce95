"""GPU: model_profiling with use_cuda=True on the four benchmark networks (MobileNetV2,
Proxyless-mobile, AtomNAS-C+, AutoNL-L) at 224x224, batch 1 and 8.

1. The counts are those of the CPU run (use_cuda=False), module for module.
2. Times: the rows of the steps run_features takes (stem convolution, every block, head
   convolution, pool, classifier Linear) are > 0; every other row, the children of the blocks
   included, is 0; the Total is their sum.
3. The Total matches an event-timed plain forward of the same input within 20 %.  Both are device
   spans from the first launch of the forward to its last: the step events telescope, so their
   sum is the profiled forward's span.  At batch 1 and 8 the host issues launches more slowly
   than the GPU runs them, so host time shows in both spans: the profiled forward's includes its
   22 event records (about 2 us of host time each on an H100 host, some 3 % of MobileNetV2's
   1.8 ms forward).  Host time is also what makes them noisy: on a quiet host the two agreed
   within 11 %, but other work on a shared host moved single medians of 10 forwards by up to 70 %.
   So the model is warmed up for half a second, and the pair is timed back to back in up to five
   rounds; the first round in which they agree passes.
4. No side effects but eval mode: parameters, buffers, BatchNorm running statistics, the
   optimizer's bf16 mirrors and state are bitwise what they were, and the TrainStep steps that
   follow (eager, then captured as a CUDA graph) are bitwise those of a run without the call.
"""
import statistics
import time

import pytest
import torch

from _cfg import build_from_cfg
from test_checkpoint_gpu import _same, _snap

pytestmark = pytest.mark.gpu
NETS = ["mobilenet_v2", "proxyless_mobile", "atomnas_c+", "autonl_l"]
TOLERANCE = 0.20
ROUNDS = 5


def _counts(model):
    return {k: (m.n_macs, m.n_params) for k, m in model.named_modules() if hasattr(m, "n_macs")}


def _plain_forward_ns(model, x, n=10):
    times = []
    with torch.no_grad():
        model(x)
        torch.cuda.synchronize()
        for _ in range(n):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            model(x)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
    return statistics.median(times) * 1e6


@pytest.mark.parametrize("batch", [1, 8])
@pytest.mark.parametrize("name", NETS)
def test_counts_and_step_times(built_lib, name, batch):
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.model_profiling import model_profiling
    model, _ = build_from_cfg(name)
    model = model.cuda().eval()
    x = torch.rand(batch, 3, 224, 224, device="cuda",
                   generator=torch.Generator("cuda").manual_seed(1))
    with torch.no_grad():
        # half a second of forwards first: the first test of a process otherwise times the
        # clocks ramping up (MobileNetV2 at batch 1 measured 1.5x its later rate)
        t_end = time.perf_counter() + 0.5
        while time.perf_counter() < t_end:
            model(x)
            torch.cuda.synchronize()
    model.train()
    fused_before = engine.EVAL_FUSED_CALLS
    n_macs, n_params = model_profiling(model, 224, 224, batch=batch, verbose=False)
    fused = engine.EVAL_FUSED_CALLS - fused_before
    got = _counts(model)
    assert not model.training

    cpu_model, _ = build_from_cfg(name)
    want = model_profiling(cpu_model, 224, 224, batch=batch, use_cuda=False, verbose=False)
    assert (n_macs, n_params) == want
    assert got == _counts(cpu_model)

    feats = list(model.features)
    blocks = feats[1:-2]
    timed = [feats[0][0], *blocks, feats[-2][0], feats[-1], model.classifier[1]]
    assert all(m.n_seconds > 0 for m in timed), [(m.name, m.n_seconds) for m in timed]
    timed_ids = {id(m) for m in timed}
    untimed = [m for m in model.modules() if hasattr(m, "name") and id(m) not in timed_ids]
    assert all(m.n_seconds == 0 for m in untimed)
    assert model.n_seconds == sum(m.n_seconds for m in timed)
    if name in ("mobilenet_v2", "proxyless_mobile"):
        # every block ran as one launch (warm-up + 10 timed forwards), its children read 0
        assert fused == 11 * len(blocks)

    # host-bound spans on a shared host: a burst of other work inflates whichever of the two is
    # being timed.  Each round times the profiled forwards and then the plain ones, back to back,
    # and the check passes on the first round in which they agree.
    diffs = []
    for r in range(ROUNDS):
        if r:
            model_profiling(model, 224, 224, batch=batch, verbose=False)
        plain = _plain_forward_ns(model, x)
        diffs.append(model.n_seconds / plain - 1)
        print("%s N=%d: rows %.3f ms, plain forward %.3f ms (%+.1f %%)"
              % (name, batch, model.n_seconds / 1e6, plain / 1e6, 100 * diffs[-1]))
        if abs(diffs[-1]) <= TOLERANCE:
            break
    assert abs(diffs[-1]) <= TOLERANCE, diffs


def _snap_all(ts, loss):
    out = _snap(ts, loss)
    for n, p in ts.model.named_parameters():
        mirror = getattr(p, "_yamb_bf16", None)
        if mirror is not None:
            out["bf16." + n] = mirror.clone()
    return out


def _run(name, profile_batch):
    from yet_another_mobilenet_series_b200.model_profiling import model_profiling
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    model, _ = build_from_cfg(name)
    model = model.cuda()
    ts = TrainStep(model, 8, image_size=224)
    g = torch.Generator().manual_seed(2)
    batches = [(torch.randn(8, 3, 224, 224, generator=g).to(torch.bfloat16),
                torch.randint(0, 1000, (8,), generator=g)) for _ in range(4)]
    snaps = [_snap_all(ts, ts(*batches[0]))]
    if profile_batch is not None:
        before = _snap_all(ts, ts.loss)
        model_profiling(model, 224, 224, batch=profile_batch, verbose=False)
        _same(_snap_all(ts, ts.loss), before)
    for b in batches[1:]:
        snaps.append(_snap_all(ts, ts(*b)))
    assert ts.graph is not None
    return snaps


@pytest.mark.parametrize("profile_batch", [1, 8])
@pytest.mark.parametrize("name", NETS)
def test_train_steps_after_profiling_are_unchanged(built_lib, name, profile_batch):
    for got, want in zip(_run(name, profile_batch), _run(name, None)):
        _same(got, want)
