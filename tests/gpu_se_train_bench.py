"""Measurement (not a test): the training step of the Squeeze-and-Excitation networks with the
default SE backward (se_bwd_reduce -> se_fc_bwd -> se_bwd_apply -> dw_bwd) against
TrainStep(fused_se=True) (se_bwd_stats -> se_fc_bwd -> se_bn_bwd_finalize -> dw_bwd_se, dz2 never
written), alternating in one process: AtomNAS-C+ at N = 256 and AutoNL-L at N = 128, 224 x 224.

For each configuration and variant: the whole step (CUDA graph replay, device events around
`--steps` steps, one sample per round, `--rounds` rounds) and, in a separate eager step with
engine.PROFILE on, the summed device time of each SE launch class (CUDA events around each launch,
launch gaps included).  Prints the card, its power limit and SM clock, read in the same run, and
one JSON line.

  python tests/gpu_se_train_bench.py --steps 10 --rounds 3"""
import argparse
import collections
import gc
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from gpu_stem_train_bench import _card, _time_steps  # noqa: E402

CONFIGS = (("atomnas_c+", 256), ("autonl_l", 128))
SE_TAGS = ("se_pool", "se_fc", "se_bwd_reduce", "se_fc_bwd", "se_bwd_apply", "se_bwd_stats",
           "se_bn_bwd_finalize", "dw_bwd", "dw_bwd_se")


def _step(name, fused, B):
    from _cfg import build_from_cfg
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    model, cfg = build_from_cfg(name)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    return TrainStep(model.cuda(), B, image_size=cfg["flags"]["image_size"], fused_se=fused)


def _se_kernels(ts, x, t):
    """{tag: summed ms} of the SE and depthwise-backward launches of one eager step."""
    from yet_another_mobilenet_series_b200 import engine
    graph, ts.graph, ts.use_graph = ts.graph, None, False
    engine.PROFILE = prof = []
    try:
        ts(x, t)
        torch.cuda.synchronize()
    finally:
        engine.PROFILE = None
        ts.graph, ts.use_graph = graph, True
    out = collections.defaultdict(float)
    for tag, _b, _f, e0, e1 in prof:
        if tag in SE_TAGS:
            out[tag] += e0.elapsed_time(e1)
    return dict(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_se_train_bench: needs a CUDA device")
    res = {"card": _card(), "steps": args.steps, "rounds": args.rounds}
    for name, B in CONFIGS:
        torch.manual_seed(0)
        x = torch.randn(B, 3, 224, 224).bfloat16()
        t = torch.randint(0, 1000, (B,))
        steps = {False: _step(name, False, B), True: _step(name, True, B)}
        for ts in steps.values():
            for _ in range(args.warmup):
                ts(x, t)
        torch.cuda.synchronize()
        times = {False: [], True: []}
        for _ in range(args.rounds):
            for fused in (False, True):
                times[fused].append(_time_steps(steps[fused], x, t, args.steps))
        res[name] = {"batch": B, "step_ms_default": times[False], "step_ms_fused_se": times[True],
                     "median_default": statistics.median(times[False]),
                     "median_fused_se": statistics.median(times[True]),
                     "se_kernels_ms_default": _se_kernels(steps[False], x, t),
                     "se_kernels_ms_fused_se": _se_kernels(steps[True], x, t),
                     "launches_per_step": {"default": steps[False].launches_per_step,
                                           "fused_se": steps[True].launches_per_step}}
        print(name, json.dumps(res[name]), flush=True)
        del steps
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
