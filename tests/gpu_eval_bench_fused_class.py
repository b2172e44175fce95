"""Eval-mode (inference) timing of the InvertedResidualChannelsFused blocks (AutoNL, AtomNAS) on
one H100: the one-launch block kernel with the Squeeze-and-Excitation gate and the non-local tail
(engine.fused_class_eval_forward) against this repo's four-launch sequence.  Driver script (not a
pytest test):

    python tests/gpu_eval_bench_fused_class.py [--config autonl_l] [--batch 256] [--iters 20]
                                               [--out FILE.json]

Per block the kernel covers: the number of C-ABI calls of the new path (1, 3 with
Squeeze-and-Excitation, 4 more with a non-local block; asserted), the summed CUDA-event time of its
kernels and of the four-launch kernels, and whether engine.FUSED_CLASS_SHAPE_RULE keeps the block on
four launches by default (both sides of the rule are timed).  Whole network: eval forward with the
shape rule, with every covered block on the new path, and with four launches everywhere.  The
card's name and power limit are read in the same run and recorded with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)


def card_name():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        if out:
            return out.splitlines()[0]
    except (OSError, subprocess.SubprocessError):
        pass
    return torch.cuda.get_device_name() + ", power limit not read"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="autonl_l", help="autonl_l | atomnas_c+ (bench.py --config)")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    import bench
    from gpu_eval_bench import kernel_time, timed
    from yet_another_mobilenet_series_b200 import engine
    dev = torch.device("cuda")
    model = bench.build_model(config=args.config).to(dev).eval()
    N = args.batch
    flush = torch.zeros(64 << 20, device=dev)
    x = torch.randn(N, 3, 224, 224, device=dev).to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last)
    res = {"config": args.config, "batch": N, "card": card_name(), "blocks": []}
    print("card:", res["card"], flush=True)

    def with_rule(on, fn):
        prev, engine.FUSED_CLASS_SHAPE_RULE = engine.FUSED_CLASS_SHAPE_RULE, on
        try:
            return fn()
        finally:
            engine.FUSED_CLASS_SHAPE_RULE = prev

    feats = list(model.features)
    h = x
    with torch.no_grad():
        for i, m in enumerate(feats):
            if hasattr(m, "expand_conv"):
                inp = h
                covered = with_rule(False, lambda: engine.fused_class_eval_supported(m, inp))
                if covered:
                    se = hasattr(m.se_op, "se_reduce")
                    nl = type(m.nl_op).__name__ != "Identity"
                    want = 1 + (2 if se else 0) + (4 if nl else 0)
                    rec = {"block": sum(hasattr(q, "use_res_connect") for q in feats[:i + 1]),
                           "shape": "%dx%dx%d -> %d (hidden %d, k %s, stride %d%s%s)" % (
                               inp.shape[1], inp.shape[2], inp.shape[3], m.output_dim,
                               sum(m.channels), list(m.kernel_sizes), m.stride,
                               ", SE" if se else "", ", non-local" if nl else ""),
                           "shape_rule_keeps_four_launches":
                               not engine.fused_class_eval_supported(m, inp)}
                    t1, n1 = with_rule(False, lambda: kernel_time(lambda: m(inp), args.iters, flush))
                    assert n1 == want, (n1, want)
                    engine.EVAL_FUSED = False
                    t4, n4 = kernel_time(lambda: m(inp), args.iters, flush)
                    engine.EVAL_FUSED = True
                    rec.update(new_path_calls=n1, new_path_us=round(t1 * 1e3, 1),
                               four_launch_us=round(t4 * 1e3, 1), four_launch_kernels=n4)
                    res["blocks"].append(rec)
                    print(rec, flush=True)
            h = m(h)

    def run():
        with torch.no_grad():
            return model(x)

    t_rule = timed(run, args.iters, flush)
    t_all = with_rule(False, lambda: timed(run, args.iters, flush))
    engine.EVAL_FUSED = False
    t_four = timed(run, args.iters, flush)
    engine.EVAL_FUSED = True
    res["network_ms"] = {"shape_rule": round(t_rule, 3),
                         "every_covered_block_new_path": round(t_all, 3),
                         "four_launch_blocks": round(t_four, 3)}
    print(json.dumps(res["network_ms"]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
