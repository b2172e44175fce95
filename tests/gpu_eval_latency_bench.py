"""Small-batch eval latency on one GPU: EvalStep.evaluate with the block kernels split over
thread-block clusters where engine.eval_cluster_size picks it, against the unsplit launch
(engine.EVAL_CLUSTER = 1), for MobileNetV2, Proxyless-mobile and AutoNL-L at N = 1 .. 64.

Per (network, N) both variants are built (one EvalStep each, its eval graph captured) and timed
in alternation for --rounds rounds:
  * evaluate_ms: one EvalStep.evaluate call on one batch (the staging copy, the graph replay and
    the host read of the metric sums), device events around it, median of --calls calls;
  * replay_ms: the captured graph alone, device events around --calls back-to-back replays.
At N = 1 it also takes per-block kernel times (engine.PROFILE: device events around every block
launch, eager forwards).  The card name and power limit are read in the same run.

  python tests/gpu_eval_latency_bench.py [--rounds 3] [--calls 50] [--out DIR]

The results go to DIR/eval_latency.json (default: a directory under the system's temporary
directory).
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

NETWORKS = ["mobilenet_v2", "proxyless_mobile", "autonl_l"]
BATCHES = [1, 2, 4, 8, 16, 64]
VARIANTS = {"rule": None, "unsplit": 1}


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return {"name": name, "power_limit_and_max_sm_clock": power,
            "sms": torch.cuda.get_device_properties(0).multi_processor_count}


def _model(name, dev):
    """The network with its BatchNorm statistics calibrated on random images by the stock-torch
    graph (an untrained AutoNL-L overflows through its non-local blocks with any others)."""
    from test_fused_class_eval_gpu import _network
    x = torch.randn(16, 3, 224, 224, generator=torch.Generator().manual_seed(4)).to(dev)
    return _network(name, 4, x).to(dev).eval()


def _evalstep(engine, model, n, cluster, batch):
    from yet_another_mobilenet_series_b200.trainer import EvalStep
    es = EvalStep(copy.deepcopy(model), n, use_graph=True)
    engine.EVAL_CLUSTER = cluster
    try:
        for _ in range(3):                   # eager warm-up, capture, replay
            es.evaluate([batch])
        assert es.phases["eval"].graph is not None
    finally:
        engine.EVAL_CLUSTER = None
    return es


def _time_evaluate(es, batch, calls):
    out = []
    for _ in range(calls):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        es.evaluate([batch])
        e1.record()
        e1.synchronize()
        out.append(e0.elapsed_time(e1))
    return statistics.median(out)


def _time_replay(es, calls):
    g = es.phases["eval"].graph
    g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / calls


def _block_times(engine, model, x, cluster, reps):
    """Median kernel time (ms) of every block launch of an eager forward, in launch order, with
    the tag of each launch (block_eval / block_eval_cluster, the SE pool passes included)."""
    engine.EVAL_CLUSTER = cluster
    runs = []
    try:
        with torch.no_grad():
            model(x)
            for _ in range(reps):
                engine.PROFILE = []
                model(x)
                torch.cuda.synchronize()
                runs.append([(t, e0.elapsed_time(e1)) for t, _, _, e0, e1 in engine.PROFILE
                             if t.startswith("block_eval")])
    finally:
        engine.PROFILE = None
        engine.EVAL_CLUSTER = None
    tags = [t for t, _ in runs[0]]
    return [(tags[i], statistics.median(r[i][1] for r in runs)) for i in range(len(tags))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--networks", default=",".join(NETWORKS))
    ap.add_argument("--batches", default=",".join(str(b) for b in BATCHES))
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "yamb_eval_latency"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import __graft_entry__ as ge
    ge.build()
    from yet_another_mobilenet_series_b200 import engine
    dev = torch.device("cuda", 0)
    card = _card()
    print("card:", card, flush=True)
    res = {"card": card, "rounds": args.rounds, "calls": args.calls, "latency": [], "blocks": {}}
    for name in args.networks.split(","):
        model = _model(name, dev)
        for n in (int(b) for b in args.batches.split(",")):
            g = torch.Generator().manual_seed(n)
            batch = (torch.randn(n, 3, 224, 224, generator=g).bfloat16(), torch.zeros(n, dtype=torch.long))
            steps = {}
            for var, cluster in VARIANTS.items():
                c0 = engine.EVAL_CLUSTER_CALLS
                steps[var] = _evalstep(engine, model, n, cluster, batch)
                steps[var].split_launches = (engine.EVAL_CLUSTER_CALLS - c0) // 2   # eager + capture
            t = {var: {"evaluate_ms": [], "replay_ms": []} for var in VARIANTS}
            for _ in range(args.rounds):
                for var, es in steps.items():
                    t[var]["evaluate_ms"].append(_time_evaluate(es, batch, args.calls))
                    t[var]["replay_ms"].append(_time_replay(es, args.calls))
            same = torch.equal(steps["rule"].logits, steps["unsplit"].logits)
            rel = float((steps["rule"].logits.float() - steps["unsplit"].logits.float()).norm() /
                        steps["unsplit"].logits.float().norm())
            row = {"network": name, "N": n, "split_launches": steps["rule"].split_launches,
                   "logits_bitwise_equal": same, "logits_rel_l2": rel}
            for var in VARIANTS:
                row[var] = {k: [round(v, 4) for v in vals] for k, vals in t[var].items()}
            res["latency"].append(row)
            print("%-16s N=%-3d split launches %3d | evaluate ms rule %s unsplit %s | replay ms rule "
                  "%s unsplit %s | logits rel %.2e" % (
                      name, n, row["split_launches"], row["rule"]["evaluate_ms"],
                      row["unsplit"]["evaluate_ms"], row["rule"]["replay_ms"],
                      row["unsplit"]["replay_ms"], rel), flush=True)
            del steps
            torch.cuda.empty_cache()
        x1 = torch.randn(1, 3, 224, 224, generator=torch.Generator().manual_seed(1)).to(dev)
        per = {var: _block_times(engine, model, x1, cluster, 20) for var, cluster in VARIANTS.items()}
        res["blocks"][name] = per
        print("%s N=1 per-block kernel ms (rule | unsplit):" % name)
        for i, ((tr, a), (tu, b)) in enumerate(zip(per["rule"], per["unsplit"])):
            print("  %2d %-22s %.4f | %-16s %.4f" % (i, tr, a, tu, b))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "eval_latency.json"), "w") as f:
        json.dump(res, f, indent=1)
    print("results:", os.path.join(args.out, "eval_latency.json"))


if __name__ == "__main__":
    main()
