"""Measurement (not a test): the training-mode stem of MobileNetV2-1.0 at N = 256, 224 x 224,
unfused (TrainStep default: stem_conv_fwd -> bn_stats -> bn_apply -> block 1 dw_fwd; backward
block 1 dw_bwd -> bn_reduce -> bn_bwd_apply -> stem_conv_wgrad) against fused
(TrainStep(fused_stem=True): stem_conv_train_fwd -> dw_fwd with the stem's BatchNorm on load;
backward dw_bwd writing dz and the stem BatchNorm's statistics -> stem_conv_train_wgrad),
alternating in one process.

For each variant: the whole step (CUDA graph replay, device events around `--steps` steps, one
sample per round, `--rounds` rounds) and, in a separate eager step with engine.PROFILE on, the
device time of each launch on the stem activation (CUDA events around each launch, launch gaps
included).  Prints the card, its power limit and SM clock, read in the same run, and one JSON line.

  python tests/gpu_stem_train_bench.py --steps 20 --rounds 3"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

# (tag, which occurrence in the step): the stem's are the first forward and the last backward
# BatchNorm launches (the head's are the others), block 1's depthwise the first dw_fwd and the
# last dw_bwd
STEM_TAGS = {False: [("stem_conv_fwd", 0), ("bn_stats", 0), ("bn_apply", 0), ("dw_fwd", 0),
                     ("dw_bwd", -1), ("bn_reduce", -1), ("bn_bwd_apply", -1),
                     ("stem_conv_wgrad", 0)],
             True: [("stem_conv_train_fwd", 0), ("dw_fwd", 0), ("dw_bwd", -1),
                    ("stem_conv_train_wgrad", 0)]}


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e


def _step(fused, B):
    from _cfg import build_from_cfg
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    model, cfg = build_from_cfg("mobilenet_v2")
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    return TrainStep(model.cuda(), B, image_size=224, fused_stem=fused)


def _time_steps(ts, x, t, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        ts(x, t)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def _stem_kernels(ts, x, t, fused):
    """{tag: ms} of the launches on the stem activation, from one eager step with engine.PROFILE."""
    from yet_another_mobilenet_series_b200 import engine
    graph, ts.graph, ts.use_graph = ts.graph, None, False
    engine.PROFILE = prof = []
    try:
        ts(x, t)
        torch.cuda.synchronize()
    finally:
        engine.PROFILE = None
        ts.graph, ts.use_graph = graph, True
    tags = [p[0] for p in prof]
    out = {}
    for tag, k in STEM_TAGS[fused]:
        idx = [i for i, g in enumerate(tags) if g == tag]
        i = idx[k]
        out[tag] = prof[i][3].elapsed_time(prof[i][4])
    out["total"] = sum(out.values())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_stem_train_bench: needs a CUDA device")
    card = _card()
    torch.manual_seed(0)
    x = torch.randn(args.batch, 3, 224, 224).bfloat16()
    t = torch.randint(0, 1000, (args.batch,))
    steps = {False: _step(False, args.batch), True: _step(True, args.batch)}
    for ts in steps.values():
        for _ in range(args.warmup):
            ts(x, t)
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for _ in range(args.rounds):
        for fused in (False, True):
            times[fused].append(_time_steps(steps[fused], x, t, args.steps))
    kern = {("fused" if f else "unfused"): _stem_kernels(steps[f], x, t, f) for f in (False, True)}
    lps = {("fused" if f else "unfused"): steps[f].launches_per_step for f in (False, True)}
    res = {"card": card, "batch": args.batch, "steps": args.steps, "rounds": args.rounds,
           "step_ms_unfused": times[False], "step_ms_fused": times[True],
           "median_unfused": statistics.median(times[False]),
           "median_fused": statistics.median(times[True]), "stem_kernels_ms": kern,
           "launches_per_step": lps}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
