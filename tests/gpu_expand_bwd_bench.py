"""GPU driver: the expand-side backward of every expanding block of MobileNetV2-1.0, per block,
run two ways (tests/expand_bwd_seq.py):

  gemms  dgrad GEMM + split-K wgrad GEMM, each forming dh1 = ca1*dz1 + cb1*h1 + cc1 in its loaders
  fused  yamb_expand_bwd: dh1 formed once, dx and dW1 from the same staged tile

The activations are real: one eager training step of the bench model per batch size records every
block's input x and its dy (dz1, h1 and the BN1-backward coefficients stay in the block's plan).
Each block runs the two sequences alternately, L2 flushed before each, on one stream, and reports
the median device time and GB/s (algorithmic bytes of engine.py's tags).  dx of the two sequences
and dW1 are compared bit for bit.
Small batches and the 14x14 / 7x7 blocks set engine.EXPAND_BWD_MIN_M.  Shapes the fused kernel
does not cover are listed as such.

  python tests/gpu_expand_bwd_bench.py [--reps 20] [--batches 256,32]
"""
import argparse
import os
import statistics
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)


def _power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            "0"], capture_output=True, text=True, timeout=20)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _record(batch, dev):
    """(plan, x [M_in, Cin], dy [M_out, Cout]) of every expanding block after one eager step."""
    import torch
    import bench
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    model = bench.build_model().to(dev)
    ts = TrainStep(model, batch, use_graph=False)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(batch, 3, 224, 224, generator=g).to(torch.bfloat16) \
        .contiguous(memory_format=torch.channels_last)
    t = torch.randint(0, 1000, (batch,), generator=g)
    ts.load(x, t)
    ts.run()
    rec = {}
    orig = engine.BlockPlan.backward

    def recording(self, x_, dy, grads):
        if self.expand:
            rec[id(self)] = (self, x_.permute(0, 2, 3, 1).reshape(self.M_in, self.Cin).clone(),
                             dy.permute(0, 2, 3, 1).reshape(self.M_out, self.Cout).clone())
        return orig(self, x_, dy, grads)

    engine.BlockPlan.backward = recording
    try:
        ts.run()
    finally:
        engine.BlockPlan.backward = orig
    torch.cuda.synchronize()
    return list(rec.values())[::-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--batches", default="256,32")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    ge.build()
    from expand_bwd_seq import ExpandBwd
    from yet_another_mobilenet_series_b200 import engine

    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)   # 256 MB > L2
    print("GPU: %s, power limit %s, %d repetitions per block and sequence"
          % (torch.cuda.get_device_name(0), _power_limit(), args.reps))
    print("engine.EXPAND_BWD_MIN_M = %d" % engine.EXPAND_BWD_MIN_M)
    all_equal = True
    for B in (int(b) for b in args.batches.split(",")):
        plans = _record(B, dev)
        print("\nN = %d" % B)
        print("%3s %8s %4s %4s %6s | %8s %8s %8s | %8s %8s | %7s %5s %6s" % (
            "blk", "M_in", "Cin", "Chid", "slabs", "dgrad", "wgrad", "gemms", "fused", "speedup",
            "GB/s g", "GB/s f", "bits"))
        tot = {"g": 0.0, "f": 0.0}
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        for bi, (p, xm, dym) in enumerate(plans):
            res = dym if p.residual else None
            eb = ExpandBwd(p.dz1, p.h1, p.bn1.ca, p.bn1.cb, p.bn1.cc, p.w_exp_bf, xm, res)
            a = eb.args()
            info = eb.nat.ExpandBwdPlanInfo()
            rc = eb.lib.yamb_expand_bwd_plan(__import__("ctypes").byref(a), 0,
                                             __import__("ctypes").byref(info))
            if rc != 0:
                print("%3d %8d %4d %4d   (not covered by yamb_expand_bwd)" % (bi + 1, p.M_in, p.Cin,
                                                                            p.Chid))
                continue
            outs = {}
            for seq in ("gemms", "fused"):
                eb.reset()
                eb.run(seq)
                torch.cuda.synchronize()
                outs[seq] = (eb.dx.clone(), eb.dw1.clone())
            eq = torch.equal(outs["gemms"][0], outs["fused"][0]) and \
                torch.equal(outs["gemms"][1], outs["fused"][1])
            all_equal = all_equal and eq
            times = {"d": [], "w": [], "f": []}
            for _ in range(args.reps):
                for seq in ("gemms", "fused"):
                    eb.reset()
                    flush.zero_()
                    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                    ev[0].record()
                    if seq == "fused":
                        eb.fused()
                        ev[1].record()
                        ev[2].record()
                    else:
                        eb.dgrad()
                        ev[1].record()
                        eb.wgrad()
                        ev[2].record()
                    torch.cuda.synchronize()
                    if seq == "fused":
                        times["f"].append(ev[0].elapsed_time(ev[1]))
                    else:
                        times["d"].append(ev[0].elapsed_time(ev[1]))
                        times["w"].append(ev[1].elapsed_time(ev[2]))
            md, mw, mf = (statistics.median(times[k]) for k in ("d", "w", "f"))
            tot["g"] += md + mw
            tot["f"] += mf
            print("%3d %8d %4d %4d %6d | %8.3f %8.3f %8.3f | %8.3f %8.2f | %7.0f %5.0f %6s" % (
                bi + 1, p.M_in, p.Cin, p.Chid, info.slabs, md, mw, md + mw, mf,
                (md + mw) / mf, eb.nbytes("gemms") / (md + mw) / 1e6, eb.nbytes("fused") / mf / 1e6,
                "same" if eq else "DIFF"))
        print("total ms  gemms %.3f  fused %.3f" % (tot["g"], tot["f"]))
    print("dx and dW1 bitwise equal in every block:", all_equal)
    return 0 if all_equal else 1


if __name__ == "__main__":
    sys.exit(main())
