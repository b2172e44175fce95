"""Gradient accumulation in TrainStep: what a step of per_gpu_batch images in micro-batches costs.

MobileNetV2-1.0 (the reference's yml), 224 x 224, bf16 input, RMSprop, one GPU, device-resident
batch (loaded once, as bench.py's device-resident timing):

  1. peak memory: torch.cuda.max_memory_allocated over construction, two eager steps, the graph
     capture and replays, each configuration alone on the device, for (per_gpu_batch,
     micro_batch) = (256, 256), (512, 256), (1024, 256), (1024, 128), (512, 512), (1024, 1024);
     a configuration that does not fit is reported as such;
  2. time: the first four built side by side and timed in alternation, ROUNDS rounds of CUDA
     events around 4096 images' worth of optimizer steps each; median ms per optimizer step,
     img/s, and time per image relative to (256, 256).

Prints one JSON line, with the card's name, power limit and max SM clock read in the same run.
Run: python tests/gpu_grad_accum_bench.py [--out result.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

TIMED = [(256, 256), (512, 256), (1024, 256), (1024, 128)]
MEMORY_ONLY = [(512, 512), (1024, 1024)]
ROUNDS, IMAGES_PER_WINDOW, WARMUP = 7, 4096, 4


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def make(per_gpu, micro):
    """A TrainStep with its batch loaded and WARMUP steps run (graph captured at the 3rd)."""
    from _cfg import build_from_cfg
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    model, _ = build_from_cfg("mobilenet_v2")
    ts = TrainStep(model.cuda(), per_gpu, micro_batch=micro)
    g = torch.Generator(device="cuda").manual_seed(per_gpu + micro)
    x = torch.randn(per_gpu, 3, 224, 224, device="cuda", generator=g).to(torch.bfloat16)
    t = torch.randint(0, 1000, (per_gpu,), device="cuda", generator=g)
    ts.load(x.contiguous(memory_format=torch.channels_last), t)
    for _ in range(WARMUP):
        ts.run()
    torch.cuda.synchronize()
    assert ts.graph is not None
    return ts


def peak_memory(per_gpu, micro):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    try:
        ts = make(per_gpu, micro)
    except torch.OutOfMemoryError:
        torch.cuda.empty_cache()
        return None
    peak = torch.cuda.max_memory_allocated() - base
    del ts
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return peak


def window(ts):
    steps = max(1, IMAGES_PER_WINDOW // ts.batch)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        ts.run()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    c = card()
    mem = {}
    for cfg in TIMED:
        mem[cfg] = peak_memory(*cfg)
    steps = {cfg: make(*cfg) for cfg in TIMED}
    for ts in steps.values():
        window(ts)
    times = {cfg: [] for cfg in TIMED}
    for r in range(ROUNDS):
        order = TIMED if r % 2 == 0 else TIMED[::-1]
        for cfg in order:
            times[cfg].append(window(steps[cfg]))
    launches = {cfg: ts.launches_per_step for cfg, ts in steps.items()}
    del steps, ts
    torch.cuda.synchronize()
    # the un-accumulated large batches last: the timings above stand if one of them does not fit
    for cfg in MEMORY_ONLY:
        mem[cfg] = peak_memory(*cfg)
    base_us = statistics.median(times[TIMED[0]]) * 1e3 / TIMED[0][0]
    rows = []
    for pg, mb in TIMED + MEMORY_ONLY:
        p = mem[(pg, mb)]
        row = {"per_gpu_batch": pg, "micro_batch": mb, "k": pg // mb,
               "peak_mem_GiB": "does not fit" if p is None else round(p / 2 ** 30, 2)}
        if (pg, mb) in times:
            ms = statistics.median(times[(pg, mb)])
            us = ms * 1e3 / pg
            row.update(ms_per_step=round(ms, 3),
                       ms_range=[round(min(times[(pg, mb)]), 3), round(max(times[(pg, mb)]), 3)],
                       img_per_s=round(pg / ms * 1e3, 1), us_per_image=round(us, 3),
                       per_image_vs_256=round(us / base_us, 4),
                       launches_per_step=launches[(pg, mb)])
        rows.append(row)
    out = {"bench": "grad_accum", "card": c, "model": "mobilenet_v2 224x224 bf16",
           "rounds": ROUNDS, "images_per_window": IMAGES_PER_WINDOW, "rows": rows}
    print(json.dumps(out), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
