"""Depthwise stage of multi-branch training blocks: per-branch launches against the grouped launch
(TrainStep(grouped_branches=True)), on AtomNAS-C and AtomNAS-C+ at N = 256.

  python tests/gpu_mb_dw_grouped_bench.py [--batch 256] [--steps 20] [--runs 3] [--out FILE]

Prints one JSON line per block kind (device time of the depthwise launches of one forward +
backward, per-branch vs grouped, from CUDA events around each launch) and one per configuration
(whole TrainStep medians, graph-replayed, the two settings alternating in one process), with the
card's name and power limit.  Writes JSON only to --out."""
import argparse
import json
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _blocks(model, hw, engine):
    out, H = [], hw
    for m in model.features:
        if hasattr(m, "expand_conv") or hasattr(m, "ops"):
            if len(engine.block_parts(m).dws) > 1:
                out.append((H, m))
            H = (H - 1) // m.stride + 1
        else:
            for conv in [c for c in m.modules() if isinstance(c, torch.nn.Conv2d)][:1]:
                H = (H - 1) // conv.stride[0] + 1
    return out


def _dw_ms(engine, m, x, dy, grouped, reps=10):
    """Median over reps of the summed device time of the depthwise launches of one fwd + bwd."""
    times = []
    for r in range(reps + 2):
        engine.TRAIN_MB_DW_GROUPED = grouped
        engine.PROFILE = []
        try:
            xg = x.clone().requires_grad_(True)
            m(xg).backward(dy)
            torch.cuda.synchronize()
            prof = engine.PROFILE
        finally:
            engine.TRAIN_MB_DW_GROUPED = False
            engine.PROFILE = None
        if r >= 2:
            times.append(sum(e0.elapsed_time(e1) for tag, _b, _f, e0, e1 in prof
                             if tag.startswith("dw_fwd") or tag.startswith("dw_bwd")))
    times.sort()
    return times[len(times) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--configs", default="atomnas_c,atomnas_c+")
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    mod = types.ModuleType("utils.config")
    mod.FLAGS = types.SimpleNamespace()
    sys.modules["utils.config"] = mod
    import __graft_entry__ as g
    g.build()
    from test_mb_dw_grouped_gpu import build_cfg
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    engine.MB_DW_SHAPE_RULE = False    # measure every kind, whatever MB_DW_FASTER lists
    card = _card()
    dev = torch.device("cuda", 0)
    results = []
    for name in args.configs.split(","):
        model, cfg = build_cfg(name)
        hw = cfg["flags"]["image_size"]
        model = model.to(dev).train()
        kinds = {}
        for H, m in _blocks(model, hw, engine):
            key = engine.mb_dw_kind(m, H, H)
            if key in kinds:
                kinds[key]["count"] += 1
                continue
            Ho = (H - 1) // m.stride + 1
            x = torch.randn(args.batch, m.input_dim, H, H, device=dev)
            dy = torch.randn(args.batch, m.output_dim, Ho, Ho, device=dev).bfloat16()
            a = _dw_ms(engine, m, x, dy, False)
            b = _dw_ms(engine, m, x, dy, True)
            kinds[key] = {"config": name, "kind": list(map(str, key)), "count": 1,
                          "per_branch_ms": round(a, 4), "grouped_ms": round(b, 4),
                          "card": card, "N": args.batch}
        for r in kinds.values():
            print(json.dumps(r))
            results.append(r)
        del model
        # whole step, graph-replayed, the two settings alternating
        steps = {}
        for grouped in (False, True):
            mdl, _ = build_cfg(name)
            steps[grouped] = TrainStep(mdl.to(dev), args.batch, image_size=hw,
                                       grouped_branches=grouped)
        gen = torch.Generator().manual_seed(0)
        x = torch.randn(args.batch, 3, hw, hw, generator=gen).bfloat16()
        t = torch.randint(0, 1000, (args.batch,), generator=gen)
        for ts in steps.values():
            for _ in range(3):
                ts(x, t)
        torch.cuda.synchronize()
        ms = {False: [], True: []}
        for _ in range(args.runs):
            for grouped, ts in steps.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    ts(x, t)
                e1.record()
                torch.cuda.synchronize()
                ms[grouped].append(e0.elapsed_time(e1) / args.steps)
        med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
        r = {"config": name, "N": args.batch, "card": card,
             "default_ms_per_step": round(med[False], 3), "grouped_ms_per_step": round(med[True], 3),
             "runs_default": [round(v, 3) for v in ms[False]],
             "runs_grouped": [round(v, 3) for v in ms[True]]}
        print(json.dumps(r))
        results.append(r)
        del steps
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
