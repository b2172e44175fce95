"""Validation timings on the GPU (not a test): python tests/gpu_eval_step_bench.py [--config NAME]

Prints the card's name, power limit and max SM clock, then, at N = --batch (256) images of 224^2,
three alternating runs of
  (a) the reference-style eager loop: model.eval() forward, cross entropy, top-k with host syncs
      per batch (common.py:67-80);
  (b) EvalStep.evaluate: graph replays, sums on the device, one sync at the end;
  (c) the stem and the head + pool, old sequence against the one-launch kernel: CUDA-event kernel
      times over many launches, algorithmic bytes and their share of the 3.35 TB/s data-sheet
      HBM3 bandwidth (the H100 SXM figure);
  (d) EvalStep.calibrate per step, eager against graph replay."""
import argparse
import copy
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def batches(n, count, classes, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(n, 3, 224, 224, generator=g).bfloat16().pin_memory(),
             torch.randint(0, classes, (n,), generator=g).pin_memory()) for _ in range(count)]


def eager_loop(model, data):
    """(a): the reference's validation loop, host syncs per batch."""
    model.eval()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        for x, t in data:
            x, t = x.cuda(non_blocking=True), t.cuda(non_blocking=True)
            out = model(x)
            loss = torch.nn.functional.cross_entropy(out, t, reduction="none")
            loss.tolist()
            pred = out.topk(5)[1].t()
            correct = pred.eq(t.view(1, -1).expand_as(pred))
            for k in (1, 5):
                (1.0 - correct[:k].float().sum(0)).cpu()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / len(data)


def timed(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n


def kernel_times(model, x, reps):
    """(c): stem and head + pool, old sequence vs one launch, CUDA events per launch."""
    from yet_another_mobilenet_series_b200 import engine, tail_ops
    feats = list(model.features)
    with torch.no_grad():
        h = x
        for layer in feats[:-2]:
            h = layer(h)
        out = {}
        for fused in (False, True, False, True):            # alternating old / new
            engine.EVAL_TAIL_FUSED = fused
            for part in ("stem", "head"):
                engine.PROFILE = []
                for _ in range(reps):
                    if part == "stem":
                        feats[0](x)
                    elif fused:
                        tail_ops.head_pool_eval(feats[-2], h)
                    else:
                        tail_ops.pw_conv_bn_act(feats[-2], h).mean((2, 3))
                torch.cuda.synchronize()
                for tag, nbytes, _, e0, e1 in engine.PROFILE:
                    rec = out.setdefault((part, fused, tag), [0.0, 0, nbytes])
                    rec[0] += e0.elapsed_time(e1)
                    rec[1] += 1
                engine.PROFILE = None
        engine.EVAL_TAIL_FUSED = False
    rows = []
    for (part, fused, tag), (ms, n, nbytes) in sorted(out.items()):
        t = ms / n * 1e-3
        rows.append("  %s %-3s %-16s %8.1f us  %7.1f MB  %5.1f %% of 3.35 TB/s" %
                    (part, "new" if fused else "old", tag, t * 1e6, nbytes / 1e6,
                     100 * nbytes / t / HBM))
    rows.append("  (the old head sequence's torch mean is not counted: it is not a launch of "
                "this library)")
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="mobilenet_v2")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--batches", type=int, default=6)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: nothing is measured without one")
    import __graft_entry__ as ge
    ge.build()
    from _cfg import build_from_cfg
    from yet_another_mobilenet_series_b200.trainer import EvalStep
    print("card:", card())
    model, _ = build_from_cfg(args.config)
    model = model.cuda().eval()
    N = args.batch
    data = batches(N, args.batches, 1000, 0)
    es = EvalStep(model, N, image_size=224)
    es_e = EvalStep(copy.deepcopy(model), N, image_size=224, use_graph=False)
    es.evaluate(data[:2])            # eager warm-up + capture
    es_e.evaluate(data[:1])
    eager_loop(model, data[:1])
    calib = data[:3]
    es.calibrate(calib)             # warm-up + capture of the calibration graph
    es_e.calibrate(calib[:1])
    for run in range(args.runs):
        a = eager_loop(model, data)
        b = timed(lambda: es.evaluate(data), len(data))
        be = timed(lambda: es_e.evaluate(data), len(data))
        dg = timed(lambda: es.calibrate(calib), len(calib))
        de = timed(lambda: es_e.calibrate(calib), len(calib))
        print("%s N=%d run %d: (a) eager loop %.2f ms/batch  (b) EvalStep graph %.2f ms/batch "
              "(eager EvalStep %.2f)  (d) calibrate graph %.2f ms/step eager %.2f ms/step"
              % (args.config, N, run, a * 1e3, b * 1e3, be * 1e3, dg * 1e3, de * 1e3))
        print("%s N=%d run %d: (c) per launch, mean over 40 launches:" % (args.config, N, run))
        print("\n".join(kernel_times(model, data[0][0].cuda(), 20)))


if __name__ == "__main__":
    main()
