"""Eval-mode (inference) timing of MobileNetV2-1.0 on one H100: the one-launch blocks
(csrc/block_eval.cu) against this repo's four-launch sequence and against the reference graph in
stock PyTorch (fp32 NCHW, autocast-bf16 channels_last).  Driver script (not a pytest test):

    python tests/gpu_eval_bench.py [--batch 256] [--iters 20] [--out gpurun_out/eval_bench.json]

Per supported block: CUDA-event time of the block alone, algorithmic bytes (x read once — twice with
the skip connection — and y written once) over that time, and the same for the four launches.
"""
import argparse
import copy
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def timed(fn, iters, flush):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.add_(1.0)                     # 256 MB write: L2 holds none of the inputs afterwards
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def kernel_time(fn, iters, flush):
    """Median over iterations of the summed device time of this repo's kernel launches inside fn
    (engine.PROFILE brackets every C-ABI launch with CUDA events): no host launch gaps."""
    from yet_another_mobilenet_series_b200 import engine
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.add_(1.0)
        engine.PROFILE = []
        fn()
        torch.cuda.synchronize()
        ts.append(sum(e0.elapsed_time(e1) for _, _, _, e0, e1 in engine.PROFILE))
        n = len(engine.PROFILE)
        engine.PROFILE = None
    ts.sort()
    return ts[len(ts) // 2], n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--config", default="mobilenet_v2",
                    help="mobilenet_v2 | proxyless_mobile | atomnas_c+ | autonl_l (bench.py --config)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.out is None:
        args.out = os.path.join(ROOT, "gpurun_out", "eval_bench%s.json" % (
            "" if args.config == "mobilenet_v2" else "_" + args.config.replace("+", "plus")))
    import __graft_entry__ as g
    g.build()
    import bench
    from oracle import torch_model as tm            # checker / context only (stock-torch graph)
    from yet_another_mobilenet_series_b200 import engine
    dev = torch.device("cuda")
    torch.backends.cudnn.benchmark = True
    model = bench.build_model(config=args.config).to(dev).eval()
    N = args.batch
    flush = torch.zeros(64 << 20, device=dev)
    x = torch.randn(N, 3, 224, 224, device=dev).to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last)
    res = {"config": args.config, "batch": N, "blocks": []}
    # ---- per block ----
    feats = list(model.features)
    h = x
    with torch.no_grad():
        for i, m in enumerate(feats):
            if hasattr(m, "use_res_connect") and hasattr(m, "channels"):
                inp = h
                rec = {"block": sum(hasattr(q, "use_res_connect") for q in feats[:i + 1]),
                       "shape": "%dx%dx%d -> %d (hidden %d, k %s, stride %d)" % (
                           inp.shape[1], inp.shape[2], inp.shape[3], m.output_dim,
                           sum(m.channels), list(m.kernel_sizes), m.stride),
                       "one_launch": bool(engine.fused_eval_supported(m, inp))}
                M_in = inp.shape[0] * inp.shape[2] * inp.shape[3]
                ho = (inp.shape[2] - 1) // m.stride + 1
                M_out = inp.shape[0] * ho * ho
                alg = 2 * (M_in * inp.shape[1] * (2 if m.use_res_connect else 1) +
                           M_out * m.output_dim)
                rec["alg_MB"] = round(alg / 1e6, 1)
                if rec["one_launch"]:
                    t1, n1 = kernel_time(lambda: m(inp), args.iters, flush)
                    assert n1 == 1, n1
                    rec["one_launch_us"] = round(t1 * 1e3, 1)
                    rec["one_launch_GBps"] = round(alg / t1 / 1e6, 1)
                engine.EVAL_FUSED = False
                t4, n4 = kernel_time(lambda: m(inp), args.iters, flush)
                engine.EVAL_FUSED = True
                rec["four_launch_us"] = round(t4 * 1e3, 1)       # kernels only, without the
                rec["four_launch_kernels"] = n4                   # torch ops that fold the BNs
                res["blocks"].append(rec)
                print(rec, flush=True)
            h = m(h)
    # ---- whole network ----
    def run(mod, inp, autocast=False):
        with torch.no_grad():
            if autocast:
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    return mod(inp)
            return mod(inp)

    t_fused = timed(lambda: run(model, x), args.iters, flush)
    engine.EVAL_FUSED = False
    t_four = timed(lambda: run(model, x), args.iters, flush)
    engine.EVAL_FUSED = True
    ref = tm.as_reference(copy.deepcopy(model)).eval()
    t_ac = timed(lambda: run(ref, x.float().contiguous(memory_format=torch.channels_last), True),
                 args.iters, flush)
    xf = x.float().contiguous()
    t_f32 = timed(lambda: run(ref, xf), max(3, args.iters // 4), flush)
    res["network_ms"] = {"one_launch_blocks": round(t_fused, 3), "four_launch_blocks": round(t_four, 3),
                         "stock_autocast_bf16_channels_last": round(t_ac, 3),
                         "stock_fp32_nchw": round(t_f32, 3)}
    res["network_img_per_s"] = {k: round(N / v * 1e3) for k, v in res["network_ms"].items()}
    print(json.dumps(res["network_ms"]), json.dumps(res["network_img_per_s"]))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
