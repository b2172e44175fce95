"""Non-local tail cost, BatchNorm vs InstanceNorm (`nl_norm`), AutoNL-L training forward+backward.

    python tests/gpu_nl_norm_bench.py [--batch 128] [--iters 5] [--rounds 2]

Builds AutoNL-L twice (the non-local norm picked through a stand-in for the reference's
utils.config FLAGS, as its train.py would), then alternates the two models `--rounds` times.  Each
round warms up and times `--iters` training iterations with engine.PROFILE on (CUDA events around
every C-ABI launch) and reports the milliseconds per iteration of every non-local launch class
(tags nl_*) summed over the 14 non-local blocks.  Prints the card name and power limit first."""
import argparse
import os
import subprocess
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + " (power limit unknown)"


def _model(nl_norm):
    flags = types.SimpleNamespace() if nl_norm is None else types.SimpleNamespace(nl_norm=nl_norm)
    mod = types.ModuleType("utils.config")
    mod.FLAGS = flags
    sys.modules["utils.config"] = mod
    try:
        from _cfg import build_from_cfg
        model, _ = build_from_cfg("autonl_l")
    finally:
        del sys.modules["utils.config"]
    g = torch.Generator().manual_seed(5)
    for m in model.modules():      # non-zero non-local norms: the branch is live
        if isinstance(m, (torch.nn.BatchNorm2d, torch.nn.InstanceNorm2d)) and m.affine:
            m.weight.data.uniform_(0.5, 1.5, generator=g)
            m.bias.data.normal_(0, 0.3, generator=g)
    return model


def _iteration(model, x, dlogits):
    logits = model(x)
    logits.backward(dlogits)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    from yet_another_mobilenet_series_b200 import engine
    dev = torch.device("cuda")
    print("card:", _card())
    models = {"BatchNorm": _model(None).to(dev).train(),
              "InstanceNorm": _model("nn.InstanceNorm").to(dev).train()}
    assert any(isinstance(m, torch.nn.InstanceNorm2d) for m in models["InstanceNorm"].modules())
    g = torch.Generator().manual_seed(0)
    x = torch.randn(a.batch, 3, 224, 224, generator=g).to(torch.bfloat16).to(dev)
    dl = torch.randn(a.batch, 1000, generator=g).to(torch.bfloat16).to(dev) * 1e-2
    results = {k: [] for k in models}
    for r in range(a.rounds):
        for name, model in models.items():
            for _ in range(2):
                _iteration(model, x, dl)
            torch.cuda.synchronize()
            engine.PROFILE = []
            for _ in range(a.iters):
                _iteration(model, x, dl)
            torch.cuda.synchronize()
            prof, engine.PROFILE = engine.PROFILE, None
            per = {}
            for tag, _, _, e0, e1 in prof:
                per[tag] = per.get(tag, 0.0) + e0.elapsed_time(e1) / a.iters
            for p in model.parameters():
                p.grad = None
            results[name].append(per)
    tags = sorted({t for rs in results.values() for per in rs for t in per if t.startswith("nl_")})
    print("AutoNL-L N=%d, ms per training iteration (forward + backward), %d iterations per "
          "round, rounds alternate" % (a.batch, a.iters))
    print("%-16s %s" % ("launch class", "  ".join("%-26s" % k for k in results)))
    for t in tags + ["nl_* total"]:
        cells = []
        for name, rs in results.items():
            if t == "nl_* total":
                vals = [sum(v for k, v in per.items() if k.startswith("nl_")) for per in rs]
            else:
                vals = [per.get(t, 0.0) for per in rs]
            cells.append("%-26s" % " / ".join("%.3f" % v for v in vals))
        print("%-16s %s" % (t, "  ".join(cells)))


if __name__ == "__main__":
    main()
