"""Multi-branch eval path against the four-launch sequence (with its _PadShadow gathers), N = 256,
224x224 inputs: per-block time of every multi-branch block of AtomNAS-C and C+ (what sets
engine.MB_SHAPE_RULE), then EvalStep.evaluate per batch with and without fused_multi_branch.

    python tests/gpu_eval_bench_multi_branch.py [--out results/eval_bench_mb.json]

Block times: CUDA events around `reps` replays of a CUDA graph of one call of the block under
no_grad, the two paths alternated five times, the median kept.  The card's name, power limit and
SM clock are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def time_block(blk, x, reps):
    """Device time of one call: the call captured in a CUDA graph (as EvalStep runs it), replayed
    `reps` times between events, so that host overhead does not count."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.no_grad(), torch.cuda.stream(s):
        for _ in range(3):
            blk(x)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            blk(x)
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import EvalStep
    from test_block_eval_mb_cpu import build, multi_branch_blocks
    dev = torch.device("cuda")
    res = {"card_before": card(), "batch": args.batch, "blocks": {}, "eval_step": {}}
    engine.MB_SHAPE_RULE = False
    for name in ("atomnas_c", "atomnas_c+"):
        model = build(name).to(dev).eval()
        blocks = multi_branch_blocks(model)
        inputs = {}
        hooks = [b.register_forward_pre_hook(lambda m, i: inputs.__setitem__(id(m), i[0]))
                 for b in blocks]
        x = torch.randn(args.batch, 3, 224, 224, device=dev)
        with torch.no_grad():
            model(x)
        for h in hooks:
            h.remove()
        rows = []
        for i, blk in enumerate(blocks):
            xin = engine.to_nhwc_bf16(inputs[id(blk)])
            t = {"mb": [], "four": []}
            for _ in range(5):
                for path in ("mb", "four"):
                    engine.EVAL_MULTI_BRANCH = path == "mb"
                    t[path].append(time_block(blk, xin, args.reps))
            engine.EVAL_MULTI_BRANCH = False
            med = {k: sorted(v)[2] for k, v in t.items()}
            row = {"block": i, "kind": list(engine.mb_kind(blk)), "shape": list(xin.shape),
                   "channels": list(blk.channels), "kernel_sizes": list(blk.kernel_sizes),
                   "mb_ms": med["mb"], "four_launch_ms": med["four"]}
            rows.append(row)
            print(name, row, flush=True)
        res["blocks"][name] = rows
        del inputs
        for flag in (False, True, False, True, False, True):
            es = EvalStep(model, args.batch, fused_multi_branch=flag)
            xb = torch.randn(args.batch, 3, 224, 224)
            tb = torch.randint(0, 1000, (args.batch,))
            batches = [(xb, tb)] * 30
            es.evaluate(batches[:5])
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            es.evaluate(batches)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / len(batches)
            res["eval_step"].setdefault(name, {}).setdefault(str(flag), []).append(ms)
            print(name, "EvalStep fused_multi_branch=%s: %.3f ms / batch" % (flag, ms), flush=True)
        del model
        torch.cuda.empty_cache()
    kinds = {}
    for name, rows in res["blocks"].items():
        for r in rows:
            k = kinds.setdefault(str(tuple(r["kind"])), {"mb_ms": 0.0, "four_launch_ms": 0.0, "n": 0})
            k["mb_ms"] += r["mb_ms"]
            k["four_launch_ms"] += r["four_launch_ms"]
            k["n"] += 1
    res["kinds"] = kinds
    for k, v in sorted(kinds.items()):
        print("kind %s: %d blocks, mb %.3f ms, four-launch %.3f ms" % (k, v["n"], v["mb_ms"],
                                                                     v["four_launch_ms"]))
    res["card_after"] = card()
    print(res["card_before"], "|", res["card_after"])
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
