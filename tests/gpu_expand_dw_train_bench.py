"""GPU benchmark of the training-mode expand + depthwise forward from x (yamb_expand_dw_train_fwd)
against the default step 2 (yamb_depthwise_fwd reading the expand GEMM's h1 back).

1. Per block kind (k, stride, H, W, Cin, Chid) of mobilenet_v2, proxyless_mobile, autonl_l and
   atomnas_c+ at the bench batch (256; 128 for autonl_l): kernel time of the fused launch and of
   dw_fwd, CUDA events over `--iters` launches each, alternating, median of 5 windows.  The expand
   GEMM runs unchanged in both steps and is not timed.
2. TrainStep ms/step of each configuration with fused_expand_dw off and on (every covered block:
   engine.EXPAND_DW_SHAPE_RULE = False), alternating, 3 rounds, CUDA graphs as bench.py runs them.

Card name, power limit and clocks are read in the same run.  Prints one summary line per kind and
per configuration; --out PATH also writes every result as JSON to PATH."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CONFIGS = {"mobilenet_v2": 256, "proxyless_mobile": 256, "autonl_l": 128, "atomnas_c+": 256}


def _card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return "nvidia-smi unavailable: %s" % e


def _kinds(name):
    """kind -> number of blocks of that kind in the configuration (input shapes at N = 1)."""
    from _cfg import build_from_cfg
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200 import engine
    model, cfg = build_from_cfg(name)
    hw = cfg["flags"]["image_size"]
    shapes = {}
    hooks = [m.register_forward_hook(lambda m, i, o, k=k: shapes.__setitem__(k, tuple(i[0].shape)))
             for k, m in enumerate(model.features)]
    with torch.no_grad():
        tm.as_reference(model).eval()(torch.zeros(1, 3, hw, hw))
    for hk in hooks:
        hk.remove()
    kinds = {}
    for k, m in enumerate(model.features):
        if hasattr(m, "expand_conv") or hasattr(m, "ops"):
            kind = engine.expand_dw_kind(m, shapes[k][2], shapes[k][3])
            if kind is not None:
                kinds[kind] = kinds.get(kind, 0) + 1
    return kinds, engine.act_code_of(model.features[1].active_fn)


def _time_kind(kind, N, act, iters):
    from test_expand_dw_train_gpu import _Bn2
    from yet_another_mobilenet_series_b200 import native as nat
    lib = nat.lib()
    k, s, H, W, Cin, Chid = kind
    g = torch.Generator().manual_seed(0)
    M, Ho, Wo = N * H * W, (H - 1) // s + 1, (W - 1) // s + 1
    Mo = N * Ho * Wo
    x = torch.randn(M, Cin, generator=g).to(torch.bfloat16).cuda()
    w1 = (torch.randn(Chid, Cin, generator=g) / Cin ** 0.5).to(torch.bfloat16).cuda()
    s1, t1 = (torch.rand(Chid, generator=g) + 0.5).cuda(), (torch.rand(Chid, generator=g) - 0.5).cuda()
    wdw = (torch.randn(Chid, 1, k, k, generator=g) / k).cuda()
    h1 = torch.empty(M, Chid, dtype=torch.bfloat16, device="cuda")
    gm = nat.Gemm()
    gm.M, gm.N, gm.K = M, Chid, Cin
    gm.A, gm.lda, gm.B, gm.ldb, gm.D, gm.ldd = x.data_ptr(), Cin, w1.data_ptr(), Cin, h1.data_ptr(), Chid
    nat.check(lib.yamb_pointwise_gemm(C.byref(gm), nat.stream_handle()))
    z = torch.empty(Mo, Chid, dtype=torch.bfloat16, device="cuda")
    z2 = torch.empty_like(z)
    bn, bn2 = _Bn2(Chid, Mo, g), _Bn2(Chid, Mo, g)
    d = nat.DwFwd()
    d.N, d.H, d.W, d.C, d.ldc, d.k, d.stride = N, H, W, Chid, Chid, k, s
    d.x, d.w, d.y = h1.data_ptr(), wdw.data_ptr(), z.data_ptr()
    d.in_scale, d.in_shift, d.in_act, d.bn = s1.data_ptr(), t1.data_ptr(), act, C.pointer(bn.s)
    a = nat.ExpandDwTrain()
    a.N, a.H, a.W, a.Cin, a.Chid, a.kernel, a.stride, a.act, a.ldh = N, H, W, Cin, Chid, k, s, act, Chid
    a.x, a.w_expand, a.bn1_scale, a.bn1_shift = x.data_ptr(), w1.data_ptr(), s1.data_ptr(), t1.data_ptr()
    a.w_dw, a.h2, a.bn = wdw.data_ptr(), z2.data_ptr(), C.pointer(bn2.s)
    calls = {"dw_fwd": lambda: lib.yamb_depthwise_fwd(C.byref(d), nat.stream_handle()),
             "fused": lambda: lib.yamb_expand_dw_train_fwd(C.byref(a), nat.stream_handle())}
    for f in calls.values():
        nat.check(f())
    torch.cuda.synchronize()
    same = torch.equal(z.view(torch.int16), z2.view(torch.int16))
    t = {n: [] for n in calls}
    for _ in range(5):
        for n, f in calls.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                f()
            e1.record()
            torch.cuda.synchronize()
            t[n].append(e0.elapsed_time(e1) * 1e3 / iters)
    med = {n: sorted(v)[len(v) // 2] for n, v in t.items()}
    return med, same


def _step_ms(name, B, fused, steps, warmup):
    from _cfg import build_from_cfg
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    model, cfg = build_from_cfg(name, seed=0)
    ts = TrainStep(model.cuda(), B, image_size=cfg["flags"]["image_size"], fused_expand_dw=fused)
    g = torch.Generator().manual_seed(1)
    hw = cfg["flags"]["image_size"]
    x = torch.randn(B, 3, hw, hw, generator=g).to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last).pin_memory()
    t = torch.randint(0, 1000, (B,), generator=g).pin_memory()
    ts.load(x, t)
    for _ in range(max(warmup, 3)):
        ts.run()
    torch.cuda.synchronize()

    def timed():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            ts.run()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps
    return ts, timed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--no-steps", action="store_true")
    ap.add_argument("--out", default=None, help="also write the results as JSON to this path")
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    from yet_another_mobilenet_series_b200 import engine
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    res = {"card": _card(), "kinds": [], "steps": {}}
    print("card:", res["card"])
    names = args.configs.split(",")
    seen = {}
    for name in names:
        kinds, act = _kinds(name)
        for kind, n in kinds.items():
            key = (kind, CONFIGS[name], act)
            if key in seen:
                continue
            med, same = _time_kind(kind, CONFIGS[name], act, args.iters)
            seen[key] = med
            row = {"config": name, "kind": list(kind), "blocks": n, "N": CONFIGS[name], "act": act,
                   "dw_fwd_us": round(med["dw_fwd"], 2), "fused_us": round(med["fused"], 2),
                   "bitwise": same}
            res["kinds"].append(row)
            print(json.dumps(row), flush=True)
    if not args.no_steps:
        engine.EXPAND_DW_SHAPE_RULE = False
        for name in names:
            B = CONFIGS[name]
            runs = {False: _step_ms(name, B, False, args.steps, args.warmup),
                    True: _step_ms(name, B, True, args.steps, args.warmup)}
            ms = {False: [], True: []}
            for _ in range(args.rounds):
                for f in (False, True):
                    ms[f].append(runs[f][1]())
            del runs
            torch.cuda.empty_cache()
            row = {"batch": B, "off_ms": [round(v, 3) for v in ms[False]],
                   "on_ms": [round(v, 3) for v in ms[True]]}
            res["steps"][name] = row
            print(name, json.dumps(row), flush=True)
    res["card_after"] = _card()
    print("card after:", res["card_after"])
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
