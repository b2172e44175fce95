"""GPU: BASELINE.json configs built from the reference's real ymls (fixture
tests/golden/model_cfgs.json) — three iterations of `TrainStep` (sm_90a kernels, CUDA graph from
the 3rd call, flat-arena RMSprop/L2/EMA) against the reference step sequence (train.py:64-114 as
restated by oracle.torch_model.RefTrainer) running the reference's stock-torch graph on the same
GPU in fp32 (truth) and under autocast-bf16 (yardstick, SURVEY.md §8c gate ii/iv).

Compared per step: the loss; after the last step: the update of every parameter tensor
(p_after - p_before, flattened over the whole network), the EMA shadows of the weights, and the
BatchNorm running statistics.  224 x 224 inputs, 1000 classes; N = 32 (N = 256 once for
MobileNetV2, the bench configuration)."""
import copy
import os

import pytest
import torch

from _cfg import build_from_cfg

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = [("mobilenet_v2", 32), ("mobilenet_v2", 256), ("proxyless_mobile", 32), ("atomnas_c+", 32),
         ("autonl_l", 32)]


def _flat(d, keys):
    return torch.cat([d[k].detach().double().flatten().cpu() for k in keys])


def _rel(a, b):
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.mark.parametrize("name,B", CASES)
def test_three_train_steps_vs_fp32_reference(built_lib, name, B):
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda")
    model, cfg = build_from_cfg(name)
    for m in model.modules():          # dropout streams differ between the three runs: off
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    fl = cfg["flags"]
    kw = dict(base_lr=fl["base_lr"], base_total_batch=fl["base_total_batch"], alpha=fl["alpha"],
              momentum=fl["momentum"], eps=fl["epsilon"], weight_decay=fl["weight_decay"],
              label_smoothing=fl["label_smoothing"], ema_decay=fl["moving_average_decay"],
              ema_base_batch=fl["moving_average_decay_base_batch"])
    ref32 = tm.RefTrainer(tm.as_reference(model).to(dev), B, **kw)
    ref16 = tm.RefTrainer(tm.as_reference(model).to(dev).to(memory_format=torch.channels_last), B,
                          autocast=torch.bfloat16, **kw)
    p0 = {k: v.detach().clone() for k, v in model.named_parameters()}
    model = model.to(dev)
    ts = TrainStep(model, B, image_size=fl["image_size"], **kw)
    g = torch.Generator().manual_seed(0)
    keys = [k for k, _ in model.named_parameters()]
    losses = {"ours": [], "fp32": [], "autocast": []}
    snaps = []
    for i in range(3):
        x = torch.randn(B, 3, 224, 224, generator=g).bfloat16()
        t = torch.randint(0, 1000, (B,), generator=g)
        xd, td = x.to(dev).float(), t.to(dev)
        l2 = float(tm.l2_loss_mnas(ref32.model, fl["weight_decay"]))
        losses["fp32"].append(ref32.step(xd, td) - l2)           # TrainStep folds L2 into the update
        l2 = float(tm.l2_loss_mnas(ref16.model, fl["weight_decay"]))
        losses["autocast"].append(ref16.step(xd.contiguous(memory_format=torch.channels_last), td) - l2)
        losses["ours"].append(float(ts(x, t)))
        snaps.append({k: v.detach().clone() for k, v in model.named_parameters()})
    torch.cuda.synchronize()
    assert ts.graph is not None                                   # the 3rd call replayed the graph
    rows = []
    try:
        # ---- loss per step ----
        rows += ["%s N=%d losses ours %s fp32 %s autocast %s" % (name, B, losses["ours"], losses["fp32"],
                                                                losses["autocast"])]
        for i in range(3):
            eo = abs(losses["ours"][i] - losses["fp32"][i])
            ea = abs(losses["autocast"][i] - losses["fp32"][i])
            assert eo <= 2.0 * ea + 5e-3 * abs(losses["fp32"][i]), rows
        # ---- parameter updates after 3 steps ----
        pt = dict(ref32.model.named_parameters())
        pa = dict(ref16.model.named_parameters())
        po = dict(model.named_parameters())
        p0f = _flat(p0, keys)
        d_t, d_a, d_o = _flat(pt, keys) - p0f, _flat(pa, keys) - p0f, _flat(po, keys) - p0f
        eo, ea = _rel(d_o, d_t), _rel(d_a, d_t)
        rows.append("update rel-L2: ours %.4f autocast %.4f" % (eo, ea))
        assert eo <= 1.3 * ea + 1e-2, rows
        # ---- EMA of the weights: (i) exactly the recurrence of utils/optim.py:53-64 applied to OUR
        #      weight trajectory, (ii) as close to the fp32 run's shadows as the autocast run's ----
        decay = fl["moving_average_decay"] ** (B / fl["moving_average_decay_base_batch"])
        worst = 0.0
        for k in keys:
            sh = p0[k].to(dev).clone()
            for step, sn in enumerate(snaps, 1):
                m = min(decay, (1.0 + step) / (10.0 + step))
                sh.mul_(m).add_(sn[k], alpha=1.0 - m)
            got = ts.opt.ema_shadow(po[k])
            worst = max(worst, float((got - sh).abs().max() / (sh.abs().max() + 1e-12)))
        rows.append("EMA recurrence max rel deviation %.2e" % worst)
        assert worst < 1e-5, rows
        s_t = _flat(ref32.ema.shadow, keys) - p0f
        s_a = _flat(ref16.ema.shadow, keys) - p0f
        s_o = torch.cat([ts.opt.ema_shadow(po[k]).detach().double().flatten().cpu() for k in keys]) - p0f
        assert _rel(s_o, s_t) <= 1.3 * _rel(s_a, s_t) + 1e-2, rows
        # ---- BatchNorm running statistics (and their EMA shadows in TrainStep) ----
        bt = dict(ref32.model.named_buffers())
        ba = dict(ref16.model.named_buffers())
        bo = dict(model.named_buffers())
        # per buffer (a global flatten is dominated by the few BatchNorms with O(100) statistics,
        # e.g. the non-local branch, whose value after three updates is itself chaotic): the
        # mean and the 90th percentile of the per-buffer errors against the autocast yardstick's
        for kind in ("running_mean", "running_var"):
            ks = [k for k in bt if k.endswith(kind)]
            eo = sorted(_rel(bo[k].double().cpu(), bt[k].double().cpu()) for k in ks)
            ea = sorted(_rel(ba[k].double().cpu(), bt[k].double().cpu()) for k in ks)
            mo, ma = sum(eo) / len(eo), sum(ea) / len(ea)
            po, pa = eo[int(0.9 * (len(eo) - 1))], ea[int(0.9 * (len(ea) - 1))]
            rows.append("%s per-buffer rel-L2: mean ours %.2e autocast %.2e; p90 ours %.2e "
                        "autocast %.2e; max ours %.2e autocast %.2e" % (kind, mo, ma, po, pa,
                                                                        eo[-1], ea[-1]))
            assert mo <= 1.5 * ma + 2e-3, rows
            assert po <= 1.5 * pa + 2e-3, rows
        nbt = [k for k in bt if k.endswith("num_batches_tracked")]
        assert all(int(bo[k]) == int(bt[k]) == 3 for k in nbt)
        sk = [n for n, b in model.named_buffers() if "running_mean" in n or "running_var" in n]
        eo = [_rel(s.detach().double().cpu(), ref32.ema.shadow[k].double().cpu())
              for s, k in zip(ts.stat_shadow, sk)]
        ea = [_rel(ref16.ema.shadow[k].double().cpu(), ref32.ema.shadow[k].double().cpu())
              for k in sk]
        mo, ma = sum(eo) / len(eo), sum(ea) / len(ea)
        rows.append("stat-shadow per-buffer mean rel-L2: ours %.2e autocast %.2e" % (mo, ma))
        assert mo <= 1.5 * ma + 2e-3, rows
    finally:
        out = os.path.join(ROOT, "gpurun_out")
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "configs_parity.txt"), "a") as f:
            f.write("\n".join(rows) + "\n")
