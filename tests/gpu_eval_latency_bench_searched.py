"""Small-batch eval latency of the searched networks on one GPU: EvalStep(small_batch=True) against
the default EvalStep() for AtomNAS-C, AtomNAS-C+ and AutoNL-L at N = 1 .. 64.

With small_batch the multi-branch blocks split their packed hidden dimension over a thread-block
cluster, and the block kinds engine.SMALL_BATCH_FASTER lists (--rule table, the default) take the
one-launch path up to their bound.  --rule off sets engine.SMALL_BATCH_RULE = False, so that every
multi-branch block and every fused-class block FUSED_CLASS_SHAPE_RULE keeps off takes it: that run
is what SMALL_BATCH_FASTER is filled from.

Per (network, N) both EvalSteps are built (their eval graphs captured) and timed in alternation for
--rounds rounds: replay_ms is the captured graph alone, device events around --calls back-to-back
replays.  launches is engine.LAUNCHES over one eager forward.  Per block whose routing the switch
changes, the block alone is captured in a CUDA graph both ways and replayed --calls times between
device events (block_us, per N), and the per-kind sums decide which kinds win at which N.  The
card's name, power limit and SM clock are read in the same run.

  python tests/gpu_eval_latency_bench_searched.py [--rule table|off] [--rounds 3] [--calls 50]
                                                  [--out DIR]

The results go to DIR/eval_latency_searched.json (default: a directory under the system's
temporary directory).
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

NETWORKS = ["atomnas_c", "atomnas_c+", "autonl_l"]
BATCHES = [1, 2, 4, 8, 16, 64]


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return {"name": name, "power_limit_sm_clock_max_sm_clock": power,
            "sms": torch.cuda.get_device_properties(0).multi_processor_count}


def _model(name, dev):
    """The network with its BatchNorm statistics calibrated on random images by the stock-torch
    graph (non-zero ZeroInitBN gammas and SE biases)."""
    import test_block_eval_mb_gpu
    import test_fused_class_eval_gpu
    x = torch.randn(16, 3, 224, 224, generator=torch.Generator().manual_seed(4)).to(dev)
    if name.startswith("atomnas"):
        return test_block_eval_mb_gpu._network(name, x)
    return test_fused_class_eval_gpu._network(name, 4, x).to(dev).eval()


def _evalstep(model, n, small, batch):
    from yet_another_mobilenet_series_b200.trainer import EvalStep
    es = EvalStep(copy.deepcopy(model), n, use_graph=True, small_batch=small)
    for _ in range(3):                       # eager warm-up, capture, replay
        es.evaluate([batch])
    assert es.phases["eval"].graph is not None
    return es


def _time_graph(g, calls):
    g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / calls


def _launches(engine, model, x, small):
    """C-ABI launches of one eager forward with EvalStep's switches."""
    engine.EVAL_SMALL_BATCH, engine.EVAL_TAIL_FUSED = small, True
    try:
        with torch.no_grad():
            l0 = engine.LAUNCHES
            model(x)
            torch.cuda.synchronize()
            return engine.LAUNCHES - l0
    finally:
        engine.EVAL_SMALL_BATCH, engine.EVAL_TAIL_FUSED = False, False


def _blocks(model):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    return [m for m in model.modules()
            if isinstance(m, (mb.InvertedResidualChannels, mb.InvertedResidualChannelsFused))]


def _block_inputs(engine, model, x):
    """The input of every block in an eager default forward (NHWC bf16)."""
    inputs = {}
    hooks = [b.register_forward_pre_hook(lambda mod, inp: inputs.__setitem__(id(mod), inp[0]))
             for b in _blocks(model)]
    try:
        with torch.no_grad():
            model(x)
    finally:
        for h in hooks:
            h.remove()
    return {k: engine.to_nhwc_bf16(v) for k, v in inputs.items()}


def _routes(engine, blk, x):
    with torch.no_grad():
        if engine.eval_supported(blk, x):
            return "one-launch"
        if engine.eval_mb_supported(blk, x):
            return "multi-branch"
    return "four-launch"


def _block_time(engine, blk, x, small, calls):
    """Device time (us) of the block alone, captured in a CUDA graph, per replay."""
    engine.EVAL_SMALL_BATCH = small
    try:
        with torch.no_grad():
            blk(x)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                blk(x)
        return 1e3 * _time_graph(g, calls)
    finally:
        engine.EVAL_SMALL_BATCH = False


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rule", choices=["table", "off"], default="table")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--networks", default=",".join(NETWORKS))
    ap.add_argument("--batches", default=",".join(str(b) for b in BATCHES))
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "yamb_eval_latency_searched"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import __graft_entry__ as ge
    ge.build()
    from yet_another_mobilenet_series_b200 import engine
    engine.SMALL_BATCH_RULE = args.rule == "table"
    dev = torch.device("cuda", 0)
    card = _card()
    print("card:", card, "| rule:", args.rule, "| SMALL_BATCH_FASTER:", engine.SMALL_BATCH_FASTER,
          flush=True)
    batches = [int(b) for b in args.batches.split(",")]
    res = {"card": card, "rule": args.rule, "table": [list(e) for e in engine.SMALL_BATCH_FASTER],
           "rounds": args.rounds, "calls": args.calls, "latency": [], "blocks": {}, "kinds": {}}
    for name in args.networks.split(","):
        model = _model(name, dev)
        per_kind = {}          # kind -> N -> [default us, small-batch us]
        res["blocks"][name] = []
        for n in batches:
            g = torch.Generator().manual_seed(n)
            batch = (torch.randn(n, 3, 224, 224, generator=g).bfloat16(), torch.zeros(n, dtype=torch.long))
            steps = {small: _evalstep(model, n, small, batch) for small in (False, True)}
            t = {small: [] for small in steps}
            for _ in range(args.rounds):
                for small, es in steps.items():
                    t[small].append(round(_time_graph(es.phases["eval"].graph, args.calls), 4))
            yd, ys = steps[False].logits.float(), steps[True].logits.float()
            rel = float((ys - yd).norm() / yd.norm())
            xd = batch[0].to(dev)
            row = {"network": name, "N": n, "default_replay_ms": t[False], "small_batch_replay_ms": t[True],
                   "default_launches": _launches(engine, steps[False].model, xd, False),
                   "small_batch_launches": _launches(engine, steps[True].model, xd, True),
                   "logits_rel_l2": rel, "logits_finite": [bool(torch.isfinite(yd).all()),
                                                          bool(torch.isfinite(ys).all())]}
            res["latency"].append(row)
            print("%-11s N=%-3d replay ms default %s small_batch %s | launches %d -> %d | logits rel %.2e"
                  " finite %s" % (name, n, t[False], t[True], row["default_launches"],
                                  row["small_batch_launches"], rel, row["logits_finite"]), flush=True)
            del steps
            # per block whose routing the switch changes
            inputs = _block_inputs(engine, model, xd.float())
            for i, blk in enumerate(_blocks(model)):
                x = inputs[id(blk)]
                r0 = _routes(engine, blk, x)
                engine.EVAL_SMALL_BATCH = True
                try:
                    r1 = _routes(engine, blk, x)
                finally:
                    engine.EVAL_SMALL_BATCH = False
                if r0 == r1 and r1 != "multi-branch":
                    continue
                kind = engine.small_batch_kind(blk)
                c0 = engine.EVAL_MB_CLUSTER_CALLS + engine.EVAL_CLUSTER_CALLS
                us = [_block_time(engine, blk, x, small, args.calls) for small in (False, True)]
                split = engine.EVAL_MB_CLUSTER_CALLS + engine.EVAL_CLUSTER_CALLS > c0
                res["blocks"][name].append({"block": i, "N": n, "kind": list(kind), "default": r0,
                                            "small_batch": r1, "split": split,
                                            "us": [round(v, 2) for v in us]})
                acc = per_kind.setdefault(kind, {}).setdefault(n, [0.0, 0.0])
                acc[0] += us[0]
                acc[1] += us[1]
                if n == 1:
                    print("  block %2d %-24s %-11s -> %-12s%s %8.2f -> %8.2f us"
                          % (i, kind, r0, r1, " split" if split else "", us[0], us[1]), flush=True)
            torch.cuda.empty_cache()
        res["kinds"][name] = {repr(k): {n: [round(v, 2) for v in p] for n, p in d.items()}
                              for k, d in per_kind.items()}
        for kind, d in sorted(per_kind.items()):
            print("  kind %-24s " % (kind,) + " ".join("N=%d %.1f->%.1f" % (n, p[0], p[1])
                                                      for n, p in sorted(d.items())), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "eval_latency_searched.json"), "w") as f:
        json.dump(res, f, indent=1)
    print("results:", os.path.join(args.out, "eval_latency_searched.json"))


if __name__ == "__main__":
    main()
