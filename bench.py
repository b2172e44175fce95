#!/usr/bin/env python
"""bench.py — images/sec of one MobileNetV2-1.0 224x224 training step (BASELINE.json metric).

  python bench.py --gpus N --steps K --warmup W            # this repo's sm_90a path
  python bench.py --impl reference --gpus N --steps K ...   # the reference's CPU path (port)
  python bench.py --impl torch_gpu --steps K ...            # context: the reference's stock-torch
                                                            # graph (cuDNN/ATen) on the same H100
  python bench.py ... --dump-outputs DIR                    # + what the last timed step computed

A step = forward + label-smoothed CE + backward + gradient all-reduce + RMSprop (with L2 decay,
EMA, bf16 repack) on one synthetic batch of 256 images per GPU (BASELINE.json configs[1];
apps/mobilenet/mobilenet_v2_mnas.yml: ReLU, BN momentum 0.01 / eps 1e-3, RMSprop alpha .9 mom .9
eps 1e-3 inside sqrt, label smoothing .1, wd 1e-5 'mnas', EMA .9999 adjusted to the batch).
One JSON line on stdout (rank 0).  With --dump-outputs DIR, rank 0 also writes what the last timed
step left to its caller as DIR/<name>.npy (float32): the loss and top-1 / top-5 fractions of the
step, every parameter of the model after its update (concatenated in named_parameters order) and
the BatchNorm running statistics.  Inputs and initial weights are seeded, so two builds can be
compared output for output.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

MBV2_ROWS = [[1, 16, 1, 1, [3]], [6, 24, 2, 2, [3]], [6, 32, 3, 2, [3]], [6, 64, 4, 2, [3]],
             [6, 96, 3, 1, [3]], [6, 160, 3, 2, [3]], [6, 320, 1, 1, [3]]]
MODEL_KW = dict(num_classes=1000, input_channel=32, last_channel=1280, width_mult=1.0,
                round_nearest=8, inverted_residual_setting=MBV2_ROWS, active_fn="nn.ReLU",
                batch_norm_momentum=0.01, batch_norm_epsilon=1e-3, dropout_ratio=0.2)


# The other BASELINE.json configurations (③ proxyless_mobile, ④ atomnas_c+, ⑤ autonl_l): model
# keywords as the reference's own yml loader resolves them (tests/golden/model_cfgs.json, written by
# oracle/make_model_cfgs.py from the reference's apps/**/*.yml).
CONFIGS = {"mobilenet_v2": ("MobileNetV2-1.0", 256), "proxyless_mobile": ("Proxyless-mobile", 256),
           "atomnas_c+": ("AtomNAS-C+ (SE, Swish)", 256), "autonl_l": ("AutoNL-L (non-local)", 128)}
_PLUGIN = {"models.mobilenet_supernet": "yet_another_mobilenet_series_b200.mobilenet_supernet",
           "models.searched_network": "yet_another_mobilenet_series_b200.searched_network"}


def build_model(seed=1995, config="mobilenet_v2"):
    import importlib
    import torch
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb, mobilenet_supernet as sup
    torch.manual_seed(seed)
    if config == "mobilenet_v2":
        model = sup.Model(**MODEL_KW, input_size=224)
    else:
        with open(os.path.join(ROOT, "tests", "golden", "model_cfgs.json")) as f:
            cfg = json.load(f)[config]
        lib = importlib.import_module(_PLUGIN[cfg["flags"]["model"]])
        model = lib.Model(**cfg["model_kwparams"], input_size=cfg["flags"]["image_size"])
    model.apply(mb.init_weights_mnas)
    return model


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.rows = []
        self.proc = None
        self.idx = gpu_index

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", "-i", str(self.idx), "--query-gpu=" + self.Q,
                 "--format=csv,noheader,nounits", "-lms", "100"],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            f = [c.strip() for c in r.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0]))
                mx.append(float(f[1]))
            except ValueError:
                continue
            for n, v in zip(names, f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "samples": len(sm), "reasons": sorted(reasons)}


def cpu_baseline(steps=3, warmup=1, batch=32, threads=None):
    """The reference's own training step on the host cores (oracle/torch_model.py port; fp32,
    N=32 — BASELINE.json configs[0]).  Bounded sample: `warmup`+`steps` steps."""
    import torch
    from oracle import torch_model as tm
    avail = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else \
        (os.cpu_count() or 1)
    model = tm.as_reference(build_model())
    trainer = tm.RefTrainer(model, batch)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(batch, 3, 224, 224, generator=g)
    t = torch.randint(0, 1000, (batch,), generator=g)
    if threads:
        cores = threads
    else:
        # "all the host threads it can use": torch's intra-op pool stops scaling (and with SMT
        # oversubscription collapses) well before 128 logical CPUs at N=32, so calibrate on one
        # step each and keep the fastest setting
        best = None
        for c in sorted({min(avail, k) for k in (8, 16, 32, 64)}):
            torch.set_num_threads(c)
            t0 = time.perf_counter()
            trainer.step(x, t)
            dt = time.perf_counter() - t0
            if best is None or dt < best[0]:
                best = (dt, c)
            if dt > 20:
                break
        cores = best[1]
    torch.set_num_threads(cores)
    for _ in range(warmup):
        trainer.step(x, t)
    times = []
    for _ in range(steps):
        t0 = time.perf_counter()
        trainer.step(x, t)
        times.append(time.perf_counter() - t0)
    times.sort()
    med = times[len(times) // 2]
    return {"value": batch / med, "unit": "img/s", "cores": cores, "kind": "port",
            "sample": "%d timed steps (median) of the reference step sequence, fp32 N=%d, after %d "
                      "warm-up; %.3f s/step" % (steps, batch, warmup, med)}, med


def host_cpu():
    """Model name and logical CPU count of the box's host (BASELINE.md §4 asks for both)."""
    name = "unknown"
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.lower().startswith("model name"):
                    name = line.split(":", 1)[1].strip()
                    break
    except OSError:
        pass
    return {"model": name, "logical_cpus": os.cpu_count(),
            "usable": len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else None}


def torch_gpu_context(batch=256, steps=5, warmup=3, device=None, config="mobilenet_v2"):
    """CONTEXT ROW (SURVEY.md §8d, BASELINE.md §4): the reference's own module graph on stock
    PyTorch kernels (cuDNN / ATen, `cudnn.benchmark = True` as train.py:133 sets it) on THIS GPU,
    the reference step sequence (Python-loop RMSprop / EMA / L2, the two host syncs of
    common.py:67-80) — fp32 NCHW exactly as the reference runs, and autocast-bf16 channels_last
    (the fastest stock configuration).  Same synthetic batch, CUDA-event timing, median."""
    import torch
    from oracle import torch_model as tm
    dev = device or torch.device("cuda", 0)
    torch.backends.cudnn.benchmark = True
    g = torch.Generator().manual_seed(0)
    x = torch.randn(batch, 3, 224, 224, generator=g).to(dev)
    t = torch.randint(0, 1000, (batch,), generator=g).to(dev)
    out = {}
    for tag, ac, cl in (("fp32_nchw", None, False), ("autocast_bf16_channels_last",
                                                     torch.bfloat16, True)):
        model = tm.as_reference(build_model(config=config)).to(dev)
        xin = x
        if cl:
            model = model.to(memory_format=torch.channels_last)
            xin = x.contiguous(memory_format=torch.channels_last)
        tr = tm.RefTrainer(model, batch, autocast=ac)
        for _ in range(warmup):
            tr.step(xin, t)
        torch.cuda.synchronize()
        full, fb = [], []
        for _ in range(steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            tr.step(xin, t)
            e1.record()
            torch.cuda.synchronize()
            full.append(e0.elapsed_time(e1))
        for _ in range(steps):      # forward + loss + backward only (no Python-loop optimizer)
            tr.opt.zero_grad()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            if ac is not None:
                with torch.autocast("cuda", dtype=ac):
                    o = model(xin).float()
            else:
                o = model(xin)
            tm.label_smooth_ce(o, t, 0.1).mean().backward()
            e1.record()
            torch.cuda.synchronize()
            fb.append(e0.elapsed_time(e1))
        full.sort()
        fb.sort()
        out[tag] = {"step_ms": round(full[len(full) // 2], 3),
                    "img_per_s": round(batch / (full[len(full) // 2] * 1e-3), 1),
                    "fwd_bwd_only_ms": round(fb[len(fb) // 2], 3)}
        del tr, model
        torch.cuda.empty_cache()
    out["what"] = ("reference module graph on stock PyTorch %s kernels (cuDNN/ATen, "
                   "cudnn.benchmark), reference step sequence incl. Python-loop RMSprop/EMA/L2 and "
                   "its 2 host syncs; N=%d; median of %d steps after %d warm-up"
                   % (torch.__version__, batch, steps, warmup))
    return out


def eval_forward_context(batch, device, config="mobilenet_v2", iters=10):
    """Supplementary (not the headline metric): model.eval() forward under no_grad on this GPU —
    the validation path of the reference (common.py:67-80).  Blocks that yamb_block_eval_fwd covers
    run in ONE launch with no intermediate in HBM (csrc/block_eval.cu); `four_launch_ms` is the same
    forward with YAMB_EVAL_FUSED off (expand GEMM, depthwise, project GEMM, BN apply per block)."""
    import torch
    from yet_another_mobilenet_series_b200 import engine
    model = build_model(config=config).to(device).eval()
    x = torch.randn(batch, 3, 224, 224, device=device).to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last)

    def timed():
        with torch.no_grad():
            for _ in range(3):
                model(x)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                model(x)
            e1.record()
            torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    c0 = engine.EVAL_FUSED_CALLS
    ms = timed()
    n_one = (engine.EVAL_FUSED_CALLS - c0) // (iters + 3)
    prev = engine.EVAL_FUSED
    engine.EVAL_FUSED = False
    try:
        ms4 = timed()
    finally:
        engine.EVAL_FUSED = prev
    return {"ms": round(ms, 3), "img_per_s": round(batch / ms * 1e3), "batch": batch,
            "one_launch_blocks": n_one, "four_launch_ms": round(ms4, 3),
            "note": "eager launches, activations of consecutive iterations exceed L2"}


def run_torch_gpu(args):
    import torch
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    ctx = torch_gpu_context(args.batch, steps=max(3, min(args.steps, 10)),
                            warmup=max(3, min(args.warmup, 5)), config=args.config)
    best = ctx["autocast_bf16_channels_last"]
    print(json.dumps({
        "impl": "torch_gpu", "metric": "images/sec", "value": best["img_per_s"], "unit": "img/s",
        "n_gpus": 1, "ms_per_step": best["step_ms"], "higher_is_better": True, "dtype": "bf16",
        "data": "synthetic", "gpu_context": ctx, "host_cpu": host_cpu(),
        "config": {"workload": "%s 224x224 training step, reference graph on stock PyTorch GPU "
                               "kernels" % CONFIGS[args.config][0], "per_gpu_batch": args.batch}}))


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    # every requested step is timed (steps x ms_per_step is the timed wall time); the CPU
    # step takes ~1-2 s, so the default 20 + 5 steps stay well under a minute
    base, med = cpu_baseline(steps=max(1, args.steps), warmup=max(1, args.warmup))
    base["host_cpu"] = host_cpu()
    line = {
        "impl": "reference", "metric": "images/sec", "value": base["value"], "unit": "img/s",
        "n_gpus": args.gpus, "steps": max(1, args.steps), "warmup": max(1, args.warmup),
        "ms_per_step": med * 1e3, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": "MobileNetV2-1.0 224x224 training step, reference CPU path "
                               "(stock torch ops, Python-loop RMSprop/EMA/L2), batch=32"},
        "cpu_baseline": base,
        "e2e": {"value": base["value"], "unit": "img/s", "h2d_bytes_per_step": 0,
                "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line))


def profile_kernels(ts, n_steps=2):
    """Per-kernel device time inside the real step: eager steps with every C-ABI launch bracketed
    by CUDA events on the launching stream; a leading device-side sleep lets the host run ahead so
    the event gaps measure kernels, not Python."""
    import torch
    from yet_another_mobilenet_series_b200 import engine
    ts_graph, ts.graph, ts.use_graph = ts.graph, None, False
    ts_world, ts.world = ts.world, 1   # rank 0 profiles alone: no collective in these extra steps
    agg = {}
    total_ms = 0.0
    try:
        for _ in range(n_steps):
            engine.PROFILE = []
            torch.cuda.synchronize()
            torch.cuda._sleep(int(2.0e8))  # ~0.1 s head start for the host
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ts.run()
            e1.record()
            torch.cuda.synchronize()
            total_ms += e0.elapsed_time(e1)
            for tag, nbytes, flops, a, b in engine.PROFILE:
                r = agg.setdefault(tag, {"ms": 0.0, "bytes": 0, "flops": 0, "launches": 0})
                r["ms"] += a.elapsed_time(b)
                r["bytes"] += nbytes
                r["flops"] += flops
                r["launches"] += 1
    finally:
        engine.PROFILE = None
        ts.graph, ts.use_graph = ts_graph, True
        ts.world = ts_world
    for r in agg.values():
        for k in ("ms", "bytes", "flops", "launches"):
            r[k] = r[k] / n_steps
    return agg, total_ms / n_steps


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d["hbm_gbs"], d.get("bf16_tflops_sustained", d["bf16_tflops"]), "measured"
    return 3350.0, 989.0, "fallback: H100 SXM data sheet (HBM3, dense BF16), not measured"


def dump_outputs(out_dir, ts, model):
    """The last timed step's results as float32 .npy files (< 64 MB for every configuration)."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    torch.cuda.synchronize()
    arrays = {"loss": ts.loss.reshape(1), "top1": ts.top1.reshape(1), "top5": ts.top5.reshape(1),
              "params": torch.cat([p.detach().float().flatten() for p in model.parameters()]),
              "bn_running_stats": torch.cat([b.detach().float().flatten() for b in ts.stat_bufs])}
    for name, t in arrays.items():
        np.save(os.path.join(out_dir, name + ".npy"), t.cpu().numpy().astype(np.float32))


def run_ours(args):
    import torch
    import torch.distributed as dist
    import __graft_entry__ as ge
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device — the sm_90a path has no CPU fallback")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    if rank == 0:
        ge.build()
    if world > 1:
        dist.barrier()
    from yet_another_mobilenet_series_b200 import engine
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    B = args.batch
    model = build_model(config=args.config).to(dev)
    if world > 1:  # rank 0's weights everywhere (reference utils/distributed.py:183-190)
        for t in model.state_dict().values():
            dist.broadcast(t, 0)
    ts = TrainStep(model, B)
    g = torch.Generator().manual_seed(rank)
    host = []
    for i in range(2):
        hx = torch.randn(B, 3, 224, 224, generator=g).to(torch.bfloat16).contiguous(
            memory_format=torch.channels_last).pin_memory()
        ht = torch.randint(0, 1000, (B,), generator=g).pin_memory()
        host.append((hx, ht))
    host_loss = torch.zeros(max(args.steps, 1), dtype=torch.float32).pin_memory()
    ts.load(*host[0])

    def sync_all():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize()

    # ---- warm-up (2 eager steps, graph capture, then replays) ----
    for _ in range(max(args.warmup, 3)):
        ts.run()
    sync_all()
    loss0 = float(ts.loss)
    # ---- timed: device-resident inputs ----
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    launches0 = engine.LAUNCHES
    sync_all()
    e0.record()
    for _ in range(args.steps):
        ts.run()
    e1.record()
    sync_all()
    ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms_total = float(ms)
    # ---- timed: end to end through TrainStep.__call__ with HOST inputs ----
    sync_all()
    e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts.load(*host[0])
    e2.record()
    for i in range(args.steps):
        ts.run()                                   # consumes the staged batch
        if i + 1 < args.steps:
            ts.load(*host[(i + 1) % 2])            # H2D of the next batch overlaps this step
        host_loss[i].copy_(ts.loss, non_blocking=True)  # D2H read of the step's result
    e3.record()
    sync_all()
    ms2 = torch.tensor([e2.elapsed_time(e3)], device=dev)
    if world > 1:
        dist.all_reduce(ms2, op=dist.ReduceOp.MAX)
    e2e_ms = float(ms2)
    clocks = sampler.stop() if rank == 0 else None
    loss_end = float(host_loss[args.steps - 1])
    if rank == 0 and args.dump_outputs:
        dump_outputs(args.dump_outputs, ts, model)
    # ---- per-kernel profile + CPU baseline (rank 0, N=1) ----
    if rank != 0:
        if world > 1:
            dist.barrier()
            dist.destroy_process_group()
        return
    agg, eager_ms = profile_kernels(ts)
    launches_per_step = ts.launches_per_step
    hbm_peak, tf_peak, peak_kind = load_peaks()
    kernels = []
    tot_k = sum(r["ms"] for r in agg.values()) or 1.0
    for tag, r in sorted(agg.items(), key=lambda kv: -kv[1]["ms"]):
        gbs = r["bytes"] / (r["ms"] * 1e-3) / 1e9 if r["ms"] > 0 else 0.0
        tfs = r["flops"] / (r["ms"] * 1e-3) / 1e12 if r["ms"] > 0 else 0.0
        kernels.append({"kernel": tag, "launches": r["launches"], "ms_per_step": round(r["ms"], 4),
                        "share": round(r["ms"] / tot_k, 4), "alg_GBps": round(gbs, 1),
                        "hbm_frac": round(gbs / hbm_peak, 4), "TFLOPs": round(tfs, 2)})
    # ---- roofline of the dominant KERNEL (launch classes that run the same __global__ function are
    # one kernel: all pw_* / head_conv_* / fc_* classes are yamb::gemm_tc_kernel) ----
    def phys(tag):
        if tag.startswith(("pw_", "head_conv", "fc_")):
            return "pw_gemm"                       # the name profiles/summarize.py gives gemm_tc_kernel
        return tag
    groups = {}
    for tag, r in agg.items():
        gk = groups.setdefault(phys(tag), {"ms": 0.0, "bytes": 0, "flops": 0, "launches": 0})
        for k in gk:
            gk[k] += r[k]
    for k in kernels:
        k["cuda_kernel"] = {"pw_gemm": "yamb::gemm_tc_kernel"}.get(phys(k["kernel"]),
                                                                  "yamb::%s_kernel" % k["kernel"])
    roofline = None
    if groups:
        name, r = max(groups.items(), key=lambda kv: kv[1]["ms"])
        traffic = None
        tpath = os.path.join(ROOT, "profiles", "traffic.json")
        if os.path.exists(tpath):
            traffic = json.load(open(tpath)).get(name)
        gbs = r["bytes"] / (r["ms"] * 1e-3) / 1e9
        tfs = r["flops"] / (r["ms"] * 1e-3) / 1e12
        roofline = {
            "kernel": {"pw_gemm": "yamb::gemm_tc_kernel (all pointwise / head / classifier GEMM "
                                  "launch classes)"}.get(name, name),
            "bound": "hbm", "achieved": round(gbs, 1), "peak": hbm_peak, "unit": "GB/s",
            "frac": round(gbs / hbm_peak, 4), "traffic": traffic, "peak_kind": peak_kind,
            "share_of_kernel_time": round(r["ms"] / tot_k, 4),
            "launches_per_step": r["launches"],
            "alg_bytes_per_launch": int(r["bytes"] / max(r["launches"], 1)),
            "avg_launch_ms": round(r["ms"] / max(r["launches"], 1), 5),
            "tensor_TFLOPs": round(tfs, 2), "tensor_frac_of_sustained_bf16": round(tfs / tf_peak, 4),
            "note": "achieved = sum of the launches' algorithmic bytes (engine.py, next to every "
                    "launch) / sum of their CUDA-event times inside real steps; traffic = mean "
                    "ncu dram bytes per launch (profiles/traffic.json)",
        }
    base = None
    gpu_ctx = None
    eval_ctx = None
    if world == 1 and not args.no_cpu_baseline:
        base, _ = cpu_baseline()
        base["host_cpu"] = host_cpu()
    if world == 1 and not args.no_gpu_context:
        del ts
        torch.cuda.empty_cache()
        gpu_ctx = torch_gpu_context(B, device=dev, config=args.config)
        try:
            eval_ctx = eval_forward_context(B, dev, config=args.config)
        except Exception as e:                      # supplementary: never takes the line down
            eval_ctx = {"error": repr(e)[:200]}
    ms_step = ms_total / args.steps
    value = B * world * args.steps / (ms_total * 1e-3)
    e2e_val = B * world * args.steps / (e2e_ms * 1e-3)
    h2d = host[0][0].numel() * 2 + host[0][1].numel() * 8
    line = {
        "metric": "images/sec", "value": value, "unit": "img/s", "n_gpus": world,
        "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": ms_step,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16",
        "data": "synthetic",
        "config": {"workload": "%s 224x224 training step (fwd+loss+bwd+all-reduce+"
                               "RMSprop/L2/EMA), bf16 activations, fp32 master weights"
                               % CONFIGS[args.config][0],
                   "per_gpu_batch": B, "global_batch": B * world, "parallelism": "dp%d" % world,
                   "l2_flush": "working set per step (>10 GB of activations at N=256) exceeds the "
                               "50 MB L2, inputs larger than L2",
                   "cuda_graph": True},
        "clocks": clocks,
        "e2e": {"value": e2e_val, "unit": "img/s", "ms_per_step": e2e_ms / args.steps,
                "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4,
                "note": "host pinned bf16 NHWC batch -> TrainStep (copy stream overlaps compute)"},
        "gpu_launches": (launches_per_step or 0) * args.steps,
        "gpu_launches_per_step": launches_per_step,
        "roofline": roofline,
        "kernels": kernels,
        "eager_profiled_step_ms": round(eager_ms, 3),
        "cpu_baseline": base,
        "gpu_context": gpu_ctx,
        "eval_forward": eval_ctx,
        "loss_first_last": [loss0, loss_end],
    }
    print(json.dumps(line))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference", "torch_gpu"])
    ap.add_argument("--batch", type=int, default=None,
                    help="per-GPU batch (default: 256; 128 for autonl_l, BASELINE.json configs)")
    ap.add_argument("--config", default="mobilenet_v2", choices=sorted(CONFIGS),
                    help="BASELINE.json model configuration (default: the headline MobileNetV2-1.0)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-gpu-context", action="store_true",
                    help="skip the stock-PyTorch-on-this-GPU context measurement")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write what the last timed step computed as DIR/<name>.npy (float32)")
    args = ap.parse_args()
    if args.batch is None:
        args.batch = CONFIGS[args.config][1]
    if args.impl == "reference":
        run_reference(args)
    elif args.impl == "torch_gpu":
        run_torch_gpu(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
