"""Measurement (not a test): the training-mode head of MobileNetV2-1.0 at N = 256, 224 x 224,
unfused (TrainStep default: head GEMM -> bn_apply -> torch mean; backward: mean backward ->
bn_reduce -> bn_bwd_apply) against fused (TrainStep(fused_tail=True): head GEMM ->
yamb_head_pool_train_fwd; backward yamb_head_pool_train_bwd), alternating in one process.

For each variant: the whole step (CUDA graph replay, device events around `--steps` steps, median
of `--rounds` rounds) and, in a separate eager pass with engine.PROFILE on, the device time per
step of the launches between the head GEMM and the head's dgrad / wgrad GEMMs, plus torch's own
kernels there (torch.profiler would be needed to see those; they are in the step time).  Prints
the card, its power limit and SM clock, and one JSON line.

  python tests/gpu_head_train_bench.py --steps 20 --rounds 3"""
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

HEAD_TAGS = ("bn_apply", "bn_reduce", "bn_bwd_apply", "head_pool_train", "head_pool_train_bwd",
             "head_conv_fwd", "head_conv_dgrad", "head_conv_wgrad")


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
    return TrainStep(model.cuda(), B, image_size=224, fused_tail=fused)


def _time_steps(ts, x, t, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        ts(x, t)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def _head_kernels(ts, x, t):
    """{tag: ms} per step of the head's launches, from one eager step with engine.PROFILE."""
    from yet_another_mobilenet_series_b200 import engine
    graph, ts.graph, ts.use_graph = ts.graph, None, False
    engine.PROFILE = prof = []
    try:
        ts(x, t)
        torch.cuda.synchronize()
    finally:
        engine.PROFILE = None
        ts.graph, ts.use_graph = graph, True
    out = {}
    # bn_apply / bn_reduce / bn_bwd_apply also serve the stem; the head's are the 1280-channel
    # ones, the last bn_apply of the forward and the first reduce / apply of the backward
    tags = [p[0] for p in prof]
    for tag in HEAD_TAGS:
        idx = [i for i, g in enumerate(tags) if g == tag]
        if not idx:
            continue
        i = idx[-1] if tag == "bn_apply" else idx[0]
        out[tag] = prof[i][3].elapsed_time(prof[i][4])
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
        raise SystemExit("gpu_head_train_bench: needs a CUDA device")
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
    kern = {("fused" if f else "unfused"): _head_kernels(steps[f], x, t) for f in (False, True)}
    res = {"card": _card(), "batch": args.batch, "steps": args.steps, "rounds": args.rounds,
           "step_ms_unfused": times[False], "step_ms_fused": times[True],
           "median_unfused": statistics.median(times[False]),
           "median_fused": statistics.median(times[True]), "head_kernels_ms": kern}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
