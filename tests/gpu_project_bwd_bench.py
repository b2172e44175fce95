"""GPU driver: the project-side backward of the 17 MobileNetV2-1.0 blocks at N = 256, per block,
formed two ways (tests/project_bwd_seq.py):

  xform  two-source dgrad + wgrad (the GEMM loaders form dh3 = ca3*dy + cb3*h3 + cc3 per tile)
  plain  bn3_bwd_apply forms dh3 once, then plain-A dgrad + wgrad (what the engine runs)

The activations are real: one eager training step of the bench model records every block's dy
(the other inputs stay in the block's plan).  Each block runs the two sequences alternately, L2
flushed before each, and reports the median device time and GB/s of every launch class, with
the algorithmic bytes of engine.py.  The outputs of the two sequences (dz2, the BN2-backward
dgamma / dbeta / ca / cb / cc and dW3) are compared bit for bit.

  python tests/gpu_project_bwd_bench.py [--reps 20] [--batch 256]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=256)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    ge.build()
    import bench
    from project_bwd_seq import ProjectBwd
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import TrainStep

    dev = torch.device("cuda")
    B = args.batch
    model = bench.build_model().to(dev)
    ts = TrainStep(model, B, use_graph=False)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, 3, 224, 224, generator=g).to(torch.bfloat16) \
        .contiguous(memory_format=torch.channels_last)
    t = torch.randint(0, 1000, (B,), generator=g)
    ts.load(x, t)
    ts.run()                                  # a real step first: BatchNorm statistics, weights
    rec = {}
    orig = engine.BlockPlan.backward

    def recording(self, x_, dy, grads):
        rec[id(self)] = (self, dy.permute(0, 2, 3, 1).reshape(self.M_out, self.Cout).clone())
        return orig(self, x_, dy, grads)

    engine.BlockPlan.backward = recording
    try:
        ts.run()
    finally:
        engine.BlockPlan.backward = orig
    torch.cuda.synchronize()
    plans = list(rec.values())[::-1]          # the backward runs the blocks last to first

    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)   # 256 MB > L2
    print("GPU: %s, power limit %s, N = %d, %d repetitions per block and sequence"
          % (torch.cuda.get_device_name(0), _power_limit(), B, args.reps))
    hdr = ("blk", "M", "Cout", "Chid", "xf dgrad", "xf wgrad", "apply", "pl dgrad", "pl wgrad",
           "xf sum", "pl sum", "apply GB/s", "bits")
    print("%3s %8s %5s %5s | %9s %9s | %9s %9s %9s | %7s %7s | %10s %5s" % hdr)
    tot = {"xf_d": 0.0, "xf_w": 0.0, "ap": 0.0, "pl_d": 0.0, "pl_w": 0.0}
    byt = {"xf_d": 0, "xf_w": 0, "ap": 0, "pl_d": 0, "pl_w": 0}
    all_equal = True
    for bi, (p, dym) in enumerate(plans):
        gamma = torch.cat([m.weight.detach().float().reshape(-1) for m in p.bn2.mods])
        bn2 = {"scale": p.bn2.scale, "shift": p.bn2.shift, "mean": p.bn2.mean,
               "invstd": p.bn2.invstd, "gamma": gamma}
        se = p.se is not None
        pb = ProjectBwd(dym, p.h3, p.h2, p.w_proj_bf, p.bn3.ca, p.bn3.cb, p.bn3.cc, bn2, p.act,
                        p.Ho * p.Wo, slices=p.bn2.slices if len(p.bn2.mods) > 1 else None,
                        gate=p.gate if se else None)
        outs = {}
        for seq in ("xform", "plain"):
            pb.reset()
            pb.run(seq)
            torch.cuda.synchronize()
            outs[seq] = pb.outputs()
        eq = all(torch.equal(outs["xform"][k], outs["plain"][k]) for k in outs["xform"])
        all_equal = all_equal and eq
        times = {k: [] for k in tot}
        for _ in range(args.reps):
            for seq in ("xform", "plain"):
                pb.reset()
                flush.zero_()
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
                ev[0].record()
                if seq == "plain":
                    pb.apply()
                ev[1].record()
                pb.dgrad(seq)
                ev[2].record()
                pb.wgrad(seq)
                ev[3].record()
                torch.cuda.synchronize()
                d, w = ev[1].elapsed_time(ev[2]), ev[2].elapsed_time(ev[3])
                if seq == "plain":
                    times["ap"].append(ev[0].elapsed_time(ev[1]))
                    times["pl_d"].append(d)
                    times["pl_w"].append(w)
                else:
                    times["xf_d"].append(d)
                    times["xf_w"].append(w)
        med = {k: statistics.median(v) for k, v in times.items()}
        M, Co, Ch = p.M_out, p.Cout, p.Chid
        b = {"xf_d": 2 * M * (2 * Co + Ch) if se else 4 * M * (Co + Ch),
             "xf_w": 2 * M * (2 * Co + Ch),
             "ap": 6 * M * Co,
             "pl_d": 2 * M * (Co + Ch) if se else 2 * M * (Co + 2 * Ch),
             "pl_w": 2 * M * (Co + Ch)}
        for k in tot:
            tot[k] += med[k]
            byt[k] += b[k]
        print("%3d %8d %5d %5d | %9.3f %9.3f | %9.3f %9.3f %9.3f | %7.3f %7.3f | %10.0f %5s"
              % (bi + 1, M, Co, Ch, med["xf_d"], med["xf_w"], med["ap"], med["pl_d"], med["pl_w"],
                 med["xf_d"] + med["xf_w"], med["ap"] + med["pl_d"] + med["pl_w"],
                 b["ap"] / med["ap"] / 1e6, "same" if eq else "DIFF"))
    print("total ms   xform: dgrad %.3f + wgrad %.3f = %.3f" % (tot["xf_d"], tot["xf_w"],
                                                               tot["xf_d"] + tot["xf_w"]))
    print("total ms   plain: apply %.3f + dgrad %.3f + wgrad %.3f = %.3f"
          % (tot["ap"], tot["pl_d"], tot["pl_w"], tot["ap"] + tot["pl_d"] + tot["pl_w"]))
    for k, name in (("xf_d", "xform dgrad"), ("xf_w", "xform wgrad"), ("ap", "bn3_bwd_apply"),
                    ("pl_d", "plain dgrad"), ("pl_w", "plain wgrad")):
        print("  %-14s %7.3f ms  %6.2f GB  %6.0f GB/s" % (name, tot[k], byt[k] / 1e9,
                                                         byt[k] / tot[k] / 1e6))
    print("outputs bitwise equal in every block:", all_equal)
    # (the time of a sequence in the training step also depends on what overlaps it: the wgrad
    # runs on a side stream there; bench.py's `kernels` block measures them in place)
    return 0 if all_equal else 1


if __name__ == "__main__":
    sys.exit(main())
