"""uint8 input path: what it costs on the GPU and what it saves on the host.

  1. stem kernels: the three uint8 entry points against their bf16 twins at N = 256, 224 x 224,
     Cout = 32 (MobileNetV2's stem), CUDA events around LAUNCHES back-to-back launches, the two
     versions alternated over ROUNDS rounds; median and spread of the per-launch time;
  2. end to end: TrainStep img/s, MobileNetV2 N = 256, from pinned host batches of uint8 (normalised
     by the stem), bf16 and fp32 (host-normalised, cast on the device);
  3. host: per-image cost of ToTensor() + Normalize() + the default collate against fast_collate
     on 224 x 224 RGB PIL images, one thread.

Prints one JSON line per part, with the card's name and power limit read in the same run.
Run: python tests/gpu_u8_input_bench.py"""
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import ctypes as C  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

N, S, COUT = 256, 224, 32
ROUNDS, LAUNCHES = 7, 20
IMAGENET = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def stem_kernels():
    from yet_another_mobilenet_series_b200 import native as nat
    lib = nat.lib()
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    u = torch.randint(0, 256, (N, S, S, 3), device=dev, dtype=torch.uint8, generator=g)
    mean = torch.tensor(IMAGENET[0], device=dev)
    std = torch.tensor(IMAGENET[1], device=dev)
    xb = u.float().div(torch.full_like(mean, 255.0)).sub(mean).div(std).to(torch.bfloat16)
    w = torch.randn(COUT, 3, 3, 3, device=dev, generator=g) * 0.3
    Ho = S // 2
    y = torch.empty(N * Ho * Ho * COUT, device=dev, dtype=torch.bfloat16)
    dh = torch.randn(N * Ho * Ho * COUT, device=dev, generator=g).to(torch.bfloat16)
    dw = torch.zeros(COUT * 27, device=dev)
    scale, shift = torch.ones(COUT, device=dev), torch.zeros(COUT, device=dev)

    def conv(x):
        a = nat.StemConv()
        a.N, a.H, a.W, a.Cout = N, S, S, COUT
        a.x, a.w, a.y, a.dh, a.dw = x.data_ptr(), w.data_ptr(), y.data_ptr(), dh.data_ptr(), dw.data_ptr()
        return a

    def u8():
        a = nat.StemConvU8()
        a.ev.conv = conv(u)
        a.ev.scale, a.ev.shift, a.ev.act = scale.data_ptr(), shift.data_ptr(), 2
        a.mean[:] = IMAGENET[0]
        a.std[:] = IMAGENET[1]
        return a

    def ev():
        e = nat.StemConvEval()
        e.conv = conv(xb)
        e.scale, e.shift, e.act = scale.data_ptr(), shift.data_ptr(), 2
        return e

    pairs = {"fwd": ((lib.yamb_stem_conv_u8_fwd, u8()), (lib.yamb_stem_conv_fwd, conv(xb))),
             "eval_fwd": ((lib.yamb_stem_conv_u8_eval_fwd, u8()), (lib.yamb_stem_conv_eval_fwd, ev())),
             "wgrad": ((lib.yamb_stem_conv_u8_wgrad, u8()), (lib.yamb_stem_conv_wgrad, conv(xb)))}
    st = torch.cuda.current_stream().cuda_stream

    def timed(fn, a):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(LAUNCHES):
            nat.check(fn(C.byref(a), st))
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) * 1e3 / LAUNCHES        # us per launch

    res = {}
    for name, ((fu, au), (fb, ab)) in pairs.items():
        timed(fu, au), timed(fb, ab)                       # warm-up
        tu, tb = [], []
        for r in range(ROUNDS):
            order = ((fu, au, tu), (fb, ab, tb)) if r % 2 == 0 else ((fb, ab, tb), (fu, au, tu))
            for fn, a, acc in order:
                acc.append(timed(fn, a))
        res[name] = {"u8_us": statistics.median(tu), "bf16_us": statistics.median(tb),
                     "u8_range_us": [min(tu), max(tu)], "bf16_range_us": [min(tb), max(tb)]}
    return res


def end_to_end(steps=30, warmup=5):
    from _cfg import build_from_cfg
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    g = torch.Generator().manual_seed(0)
    u = torch.randint(0, 256, (N, S, S, 3), dtype=torch.uint8, generator=g)
    t = torch.randint(0, 1000, (N,), generator=g).pin_memory()
    mean, std = torch.tensor(IMAGENET[0]), torch.tensor(IMAGENET[1])
    f32 = u.float().div(255).sub(mean).div(std)
    inputs = {"uint8": (u.permute(0, 3, 1, 2).pin_memory(), torch.uint8),
              "bf16": (f32.to(torch.bfloat16).permute(0, 3, 1, 2).pin_memory(), torch.bfloat16),
              "fp32": (f32.permute(0, 3, 1, 2).pin_memory(), torch.bfloat16)}
    res = {}
    for name, (x, dtype) in inputs.items():
        model, _ = build_from_cfg("mobilenet_v2")
        model = model.cuda()
        kw = {"input_norm": IMAGENET} if dtype == torch.uint8 else {}
        ts = TrainStep(model, N, input_dtype=dtype, **kw)
        for _ in range(warmup):
            ts(x, t)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            ts(x, t)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        res[name] = {"img_per_s": N * steps / dt, "ms_per_step": 1e3 * dt / steps,
                     "h2d_bytes_per_image": x[0].numel() * x.element_size()}
        del ts, model
        torch.cuda.empty_cache()
    return res


def host_cost(n=64, reps=5):
    from PIL import Image
    from torch.utils.data import default_collate
    from torchvision import transforms
    from yet_another_mobilenet_series_b200.dataflow import fast_collate
    torch.set_num_threads(1)
    rng = np.random.default_rng(0)
    imgs = [Image.fromarray(rng.integers(0, 256, (S, S, 3), dtype=np.uint8)) for _ in range(n)]
    tf = transforms.Compose([transforms.ToTensor(), transforms.Normalize(*IMAGENET)])

    def ref():
        return default_collate([(tf(im), 0) for im in imgs])

    def fast():
        return fast_collate([(im, 0) for im in imgs])

    out = {}
    for name, fn in (("totensor_normalize_collate", ref), ("fast_collate", fast)):
        fn()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            fn()
            ts.append(time.perf_counter() - t0)
        out[name + "_us_per_image"] = 1e6 * statistics.median(ts) / n
    return out


def main():
    import __graft_entry__ as g
    g.build()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    c = card()
    print(json.dumps({"part": "stem_kernels", "card": c, "N": N, "size": S, "Cout": COUT,
                      **stem_kernels()}), flush=True)
    print(json.dumps({"part": "end_to_end", "card": c, "N": N, **end_to_end()}), flush=True)
    print(json.dumps({"part": "host", "card": c, "threads": 1, **host_cost()}), flush=True)


if __name__ == "__main__":
    main()
