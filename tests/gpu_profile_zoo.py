"""model_profiling tables of the four benchmark networks (bench.py's configurations: MobileNetV2,
Proxyless-mobile, AtomNAS-C+, AutoNL-L, 224x224) at batch 1 and 256, on one GPU.

For each (network, batch), after half a second of warm-up forwards: the full table
(`model_profiling(..., use_cuda=True)`, every time the median device time of 10 forwards) and,
for comparison, the median device time of 10 plain event-timed forwards of the same input.  The
card's name, power limit and max SM clock are read in the same run.

  python tests/gpu_profile_zoo.py [--batches 1 256] [--out DIR]

Prints a summary per (network, batch); writes every table to DIR/profile_<network>_<batch>.txt
and the summary to DIR/profile_zoo.json (default DIR: one under the system's temporary
directory).
"""
import argparse
import json
import logging
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


class _Lines(logging.Handler):
    def __init__(self):
        super().__init__()
        self.lines = []

    def emit(self, record):
        self.lines.append(record.getMessage())


def plain_forward_ms(model, x, n=10):
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
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 256])
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "yamb_profile_zoo"))
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    import bench
    from yet_another_mobilenet_series_b200.model_profiling import model_profiling
    os.makedirs(args.out, exist_ok=True)
    handler = _Lines()
    root = logging.getLogger()
    root.addHandler(handler)
    root.setLevel(logging.INFO)
    result = {"card": card(), "runs": []}
    print("card:", result["card"])
    for config in bench.CONFIGS:
        for n in args.batches:
            model = bench.build_model(config=config).cuda().eval()
            x = torch.rand(n, 3, 224, 224, device="cuda",
                           generator=torch.Generator("cuda").manual_seed(0))
            with torch.no_grad():       # half a second of forwards: clocks and caches settle
                t_end = time.perf_counter() + 0.5
                while time.perf_counter() < t_end:
                    model(x)
                    torch.cuda.synchronize()
            handler.lines = []
            n_macs, n_params = model_profiling(model, 224, 224, batch=n)
            table = handler.lines
            with open(os.path.join(args.out, "profile_%s_%d.txt" % (config, n)), "w") as f:
                f.write("\n".join(table) + "\n")
            plain = plain_forward_ms(model, x)
            timed = [(m.name, m.n_seconds) for m in model.modules()
                     if hasattr(m, "name") and m.n_seconds]
            run = {"config": config, "batch": n, "n_macs": n_macs, "n_params": int(n_params),
                   "rows_ms": model.n_seconds / 1e6, "plain_forward_ms": plain,
                   "blocks_ms": sum(t for name, t in timed if "Inverted" in name) / 1e6}
            result["runs"].append(run)
            print("%-17s N=%-4d MACs %s  params %s  rows %.3f ms  blocks %.3f ms  plain forward "
                  "%.3f ms" % (config, n, "{:,}".format(n_macs), "{:,}".format(n_params),
                               run["rows_ms"], run["blocks_ms"], plain))
            del model
            torch.cuda.empty_cache()
    with open(os.path.join(args.out, "profile_zoo.json"), "w") as f:
        json.dump(result, f, indent=1)
    root.removeHandler(handler)


if __name__ == "__main__":
    main()
