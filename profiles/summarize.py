"""Turn the ncu CSV exports brought back from the GPU box (gpurun_out/<round>_*.csv) into the
committed evidence under profiles/:
  <round>_launches_step.csv      every launch of one training step: time + DRAM bytes (trimmed)
  <round>_step_summary.md        per-kernel-class totals and shares of the step
  <round>_ncu_b3_summary.md      --set full highlights of one block's kernels
  traffic.json                   measured DRAM bytes per launch per kernel class (bench.py reads it)
Usage: python profiles/summarize.py r01
"""
import csv
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "profiles")
SRC = os.path.join(ROOT, "gpurun_out")


def tag_of(name, prev_gemm=[0]):
    if "dw_fwd_kernel" in name:
        return "dw_fwd"
    if "dw_bwd_kernel" in name:
        return "dw_bwd"
    if "gemm_tc_kernel" in name:
        return "pw_gemm"
    for k in ("bn_bwd_apply", "bn_stats", "bn_apply", "bn_reduce", "se_pool", "se_bwd_reduce", "se_bwd_apply", "rmsprop",
              "ema_kernel", "cast_bf16", "stem_fwd", "stem_wgrad", "softmax_ce_fwd", "softmax_ce_bwd",
              "colsum_bf16", "se_fc_fwd", "se_fc_bwd_sample", "se_fc_bwd_param", "nl_gram", "nl_rowmat"):
        if k in name:
            return k
    return "torch:" + re.sub(r"<.*", "", name.replace("void ", ""))[:48]


def read_ncu_csv(path):
    rows = list(csv.reader(open(path)))
    hi = next(i for i, r in enumerate(rows) if r and r[0] == "ID")
    body = rows[hi + 1:]
    units = None
    if body and body[0] and not body[0][0].strip().isdigit():   # wide format: a units row follows
        units, body = body[0], body[1:]
    read_ncu_csv.units = units
    return rows[hi], body


def step(rnd):
    path = os.path.join(SRC, rnd + "_launches_step.csv")
    hdr, body = read_ncu_csv(path)
    col = {h: i for i, h in enumerate(hdr)}
    # long format: one row per (launch, metric)
    launches = {}
    for r in body:
        if len(r) < len(hdr):
            continue
        lid = int(r[col["ID"]])
        d = launches.setdefault(lid, {"name": r[col["Kernel Name"]]})
        d[r[col["Metric Name"]]] = (float(r[col["Metric Value"]].replace(",", "")),
                                    r[col["Metric Unit"]])
    def to_bytes(v):
        val, unit = v
        mult = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1)
        return val * mult
    def to_us(v):
        val, unit = v
        return val * {"ns": 1e-3, "us": 1, "ms": 1e3, "s": 1e6}.get(unit, 1)
    agg, lines = {}, []
    for lid in sorted(launches):
        d = launches[lid]
        t = to_us(d["gpu__time_duration.sum"])
        rd = to_bytes(d["dram__bytes_read.sum"])
        wr = to_bytes(d["dram__bytes_write.sum"])
        tg = tag_of(d["name"])
        a = agg.setdefault(tg, {"us": 0.0, "dram": 0.0, "n": 0})
        a["us"] += t
        a["dram"] += rd + wr
        a["n"] += 1
        lines.append((lid, tg, d["name"][:70], round(t, 2), int(rd), int(wr)))
    with open(os.path.join(OUT, rnd + "_launches_step.csv"), "w") as f:
        w = csv.writer(f)
        w.writerow(["id", "class", "kernel", "time_us", "dram_read_bytes", "dram_write_bytes"])
        w.writerows(lines)
    tot = sum(a["us"] for a in agg.values())
    ours = sum(a["us"] for k, a in agg.items() if not k.startswith("torch:"))
    with open(os.path.join(OUT, rnd + "_step_summary.md"), "w") as f:
        f.write("# %s — one eager MobileNetV2-1.0 training step under ncu (N=256)\n\n" % rnd)
        f.write("`ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum "
                "--clock-control none` over `tests/gpu_step_once.py` (serialised, cold caches: "
                "use the SHARES).  %d launches, %.2f ms of kernel time, %.1f %% in this repo's "
                "kernels.\n\n" % (len(lines), tot / 1e3, 100 * ours / tot))
        f.write("| class | launches | time ms | share | DRAM GB | DRAM GB/s |\n|---|---|---|---|---|---|\n")
        for k, a in sorted(agg.items(), key=lambda kv: -kv[1]["us"])[:30]:
            f.write("| %s | %d | %.3f | %.1f %% | %.3f | %.0f |\n" % (
                k, a["n"], a["us"] / 1e3, 100 * a["us"] / tot, a["dram"] / 1e9,
                a["dram"] / (a["us"] * 1e-6) / 1e9 if a["us"] else 0))
    traffic = {k: a["dram"] / a["n"] for k, a in agg.items() if not k.startswith("torch:")}
    json.dump(traffic, open(os.path.join(OUT, "traffic.json"), "w"), indent=1)
    print("step:", len(lines), "launches", round(tot / 1e3, 2), "ms")


BLOCK_DESC = {"b1": "b1 (32->16, no expand, 112x112)", "b3": "b3 (24->144->24, 56x56)",
              "b8": "b8 (64->384->64, 14x14)", "b15": "b15 (160->960->160, 7x7)",
              "b2": "b2 (16->96->24, 112x112 -> 56x56)"}


def block(rnd, name="b3"):
    path = os.path.join(SRC, "%s_ncu_%s_raw.csv" % (rnd, name))
    if not os.path.exists(path):
        return
    hdr, body = read_ncu_csv(path)
    units = read_ncu_csv.units or [""] * len(hdr)
    col = {h: i for i, h in enumerate(hdr)}

    def cell(r, key):
        if key not in col:
            return "-"
        v, u = r[col[key]], units[col[key]]
        scale = {"Gbyte": 1e3, "Mbyte": 1.0, "Kbyte": 1e-3, "byte": 1e-6}
        if u in scale:  # bytes -> MB
            return "%.1f" % (float(v.replace(",", "")) * scale[u])
        if u in ("us", "ns", "ms"):
            return "%.1f" % (float(v.replace(",", "")) * {"us": 1, "ns": 1e-3, "ms": 1e3}[u])
        try:
            return "%.1f" % float(v.replace(",", ""))
        except ValueError:
            return v
    want = [("gpu__time_duration.sum", "time us"), ("dram__bytes_read.sum", "dram rd MB"),
            ("dram__bytes_write.sum", "dram wr MB"),
            ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram %"),
            ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor %"),
            ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue %"),
            ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps %"),
            ("sm__warps_active.avg.per_cycle_active", "warps/cycle"),
            ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "stall long_sb"),
            ("smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "stall barrier"),
            ("smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "stall short_sb"),
            ("launch__registers_per_thread", "regs"), ("launch__grid_size", "grid"),
            ("lts__t_sector_hit_rate.pct", "L2 hit %")]
    with open(os.path.join(OUT, "%s_ncu_%s_summary.md" % (rnd, name)), "w") as f:
        f.write("# %s — ncu --set full, block %s, N=256, forward+backward\n\n" %
                (rnd, BLOCK_DESC.get(name, name)))
        f.write("(stall columns: warps stalled per issue-active cycle, ncu's "
                "`smsp__average_warps_issue_stalled_*_per_issue_active.ratio`)\n\n")
        f.write("| kernel | " + " | ".join(w[1] for w in want) + " |\n|---|" + "---|" * len(want) + "\n")
        for r in body:
            if len(r) < len(hdr) or "yamb::" not in r[col["Kernel Name"]]:
                continue
            name = re.sub(r"\(.*", "", r[col["Kernel Name"]].replace("void yamb::", ""))[:44]
            f.write("| %s | " % name + " | ".join(cell(r, w[0]) for w in want) + " |\n")
    print("block summary written")


def eval_blocks(rnd, names=("b1", "b2", "b3", "b8", "b15")):
    """ncu --set full of the one-launch eval-mode block kernel (csrc/block_eval.cu) on several
    MobileNetV2 blocks at N = 256 (tests/gpu_profile_block.py with YAMB_PROFILE_EVAL=1)."""
    path = os.path.join(SRC, "%s_ncu_eval_raw.csv" % rnd)
    if not os.path.exists(path):
        return
    hdr, body = read_ncu_csv(path)
    units = read_ncu_csv.units or [""] * len(hdr)
    col = {h: i for i, h in enumerate(hdr)}

    def num(r, key):
        v, u = r[col[key]], units[col[key]]
        x = float(v.replace(",", ""))
        scale = {"Gbyte": 1e3, "Mbyte": 1.0, "Kbyte": 1e-3, "byte": 1e-6, "us": 1, "ns": 1e-3, "ms": 1e3}
        return x * scale.get(u, 1.0)
    want = [("gpu__time_duration.sum", "time us"), ("dram__bytes_read.sum", "dram rd MB"),
            ("dram__bytes_write.sum", "dram wr MB"),
            ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram %"),
            ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor %"),
            ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue %"),
            ("sm__warps_active.avg.per_cycle_active", "warps/cycle"),
            ("smsp__inst_executed.sum", "warp instr"),
            ("smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "stall barrier"),
            ("smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "stall wait"),
            ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "stall long_sb"),
            ("smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "stall short_sb"),
            ("launch__registers_per_thread", "regs"), ("launch__grid_size", "grid"),
            ("launch__shared_mem_per_block_dynamic", "smem KB"),
            ("lts__t_sector_hit_rate.pct", "L2 hit %")]
    rows = [r for r in body if len(r) >= len(hdr) and "block_eval_kernel" in r[col["Kernel Name"]]]
    with open(os.path.join(OUT, "%s_ncu_eval_summary.md" % rnd), "w") as f:
        f.write("# %s — ncu --set full, eval-mode block in ONE launch (`yamb::block_eval_kernel`), "
                "N=256\n\n" % rnd)
        f.write("`YAMB_PROFILE_EVAL=1 ncu --set full --clock-control none -k regex:block_eval python "
                "tests/gpu_profile_block.py %s` (one profiled launch per block after two warm-up "
                "iterations; serialised, cold caches).  Algorithmic bytes of a block: x read once "
                "(twice with the skip connection), y written once — the hidden tensors never reach "
                "HBM, so `dram rd + wr` here IS the block's whole traffic.\n\n" % " ".join(names))
        f.write("| block | " + " | ".join(w[1] for w in want) + " |\n|---|" + "---|" * len(want) + "\n")
        for name, r in zip(names, rows):
            cells = []
            for key, _ in want:
                if key not in col:
                    cells.append("-")
                    continue
                x = num(r, key)
                cells.append("%.0f" % x if x >= 1000 else "%.2f" % x if x < 10 else "%.1f" % x)
            f.write("| %s | " % BLOCK_DESC.get(name, name) + " | ".join(cells) + " |\n")
    print("eval block summary written:", len(rows), "kernels")


def bench_launches(rnd):
    """ncu launch list of `python bench.py --steps 2 --warmup 1` itself
    (`ncu --metrics gpu__time_duration.sum --clock-control none -c 1600 --csv`): trimmed CSV +
    per-class shares of the complete eager steps it contains (between two rmsprop launches)."""
    path = os.path.join(SRC, rnd + "_launches_bench.csv")
    if not os.path.exists(path):
        return
    hdr, body = read_ncu_csv(path)
    col = {h: i for i, h in enumerate(hdr)}
    rows = []
    for r in body:
        if len(r) < len(hdr) or r[col["Metric Name"]] != "gpu__time_duration.sum":
            continue
        unit = r[col["Metric Unit"]]
        t = float(r[col["Metric Value"]].replace(",", "")) * {"ns": 1e-3, "us": 1, "ms": 1e3}.get(unit, 1)
        rows.append((int(r[col["ID"]]), r[col["Kernel Name"]], t))
    with open(os.path.join(OUT, rnd + "_launches_bench.csv"), "w") as f:
        w = csv.writer(f)
        w.writerow(["id", "class", "kernel", "time_us"])
        for lid, name, t in rows:
            w.writerow([lid, tag_of(name), name[:70], round(t, 2)])
    ends = [i for i, (_, n, _) in enumerate(rows) if "rmsprop" in n]
    agg, nsteps = {}, 0
    for a, b in zip(ends[:-1], ends[1:]):
        nsteps += 1
        for _, n, t in rows[a + 1:b + 1]:
            g = agg.setdefault(tag_of(n), [0, 0.0])
            g[0] += 1
            g[1] += t
    if not nsteps:
        return
    tot = sum(v[1] for v in agg.values())
    with open(os.path.join(OUT, rnd + "_launches_bench_summary.md"), "w") as f:
        f.write("# %s — kernel launches of `python bench.py --steps 2 --warmup 1` under ncu\n\n" % rnd)
        f.write("`ncu --metrics gpu__time_duration.sum --clock-control none -c 1600 --csv` -> "
                "`%s_launches_bench.csv` (%d launches).  Below: the %d complete steps between "
                "consecutive `rmsprop` launches, %.2f ms of kernel time per step (serialised, "
                "cold-cache: compare the SHARES with the `kernels` block of the bench line).\n\n"
                % (rnd, len(rows), nsteps, tot / nsteps / 1e3))
        f.write("| class | launches/step | ms/step | share |\n|---|---|---|---|\n")
        for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:28]:
            f.write("| %s | %.1f | %.3f | %.1f %% |\n" % (k, n / nsteps, t / nsteps / 1e3, 100 * t / tot))
    print("bench launch summary written:", nsteps, "steps")


if __name__ == "__main__":
    rnd = sys.argv[1] if len(sys.argv) > 1 else "r01"
    step(rnd)
    for b in ("b1", "b2", "b3", "b8", "b15"):
        block(rnd, b)
    bench_launches(rnd)
    eval_blocks(rnd)
