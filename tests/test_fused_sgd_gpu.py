"""GPU: the fused flat-arena SGD (`yamb_sgd_step`) and the SGD recipe of apps/mobilenet/default.yml.

  * the kernel against the live reference's sequences (tests/golden/optim_sgd.pt): parameters
    <= 2e-6 rel-L2 over 12 steps, momentum buffers <= 1e-5 (the gates of test_optimizer_gpu.py);
  * several tensors with the 'slimmable' L2 folded in, the EMA warm-up rule, grad_scale and
    nesterov against the oracle (tests/sgd_oracle.py), bf16 mirror exact;
  * state_dict interchange with torch.optim.SGD in both directions;
  * gradless parameters and gradients that left the arena;
  * three TrainStep steps with the default.yml hyper-parameters against the reference step sequence
    (tests/sgd_oracle.RefTrainer) in fp32 (truth) and autocast-bf16 (yardstick), by the rule of
    test_configs_gpu.py; the same for RMSprop with the 'slimmable' L2;
  * graph replay and eager give the same bits with SGD."""
import copy
import os

import numpy as np
import pytest
import torch

import sgd_oracle as so
from _cfg import build_from_cfg, load_cfgs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# apps/mobilenet/default.yml:14-31 (optimizer: sgd)
BASE_LR = 0.5              # :21 base_lr
BASE_TOTAL_BATCH = 1024    # :22 base_total_batch
MOMENTUM = 0.9             # :15 momentum
WEIGHT_DECAY = 1e-4        # :16 weight_decay (:17 weight_decay_method: slimmable)
NESTEROV = True            # :18 nesterov
LABEL_SMOOTHING = 0.0      # :27 label_smoothing
EMA_DECAY = 0.0            # :30 moving_average_decay (0: no EMA)


def _rel(a, b):
    a = a.detach().double().cpu().numpy() if torch.is_tensor(a) else np.asarray(a, np.float64)
    b = b.detach().double().cpu().numpy() if torch.is_tensor(b) else np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))


@pytest.mark.parametrize("tag", list(so.SGD_CASES))
def test_sgd_vs_golden(built_lib, golden_dir, tag):
    from yet_another_mobilenet_series_b200.fused_sgd import SGD
    rec = so.load_golden()[tag]
    names = list(rec["params"])
    ps = {k: torch.nn.Parameter(rec["params"][k]["p0"].clone().cuda()) for k in names}
    opt = SGD(list(ps.values()), **rec["kw"])
    for i in range(so.STEPS):
        opt.zero_grad()
        for k, p in ps.items():
            s = rec["params"][k]
            if bool(s["has_grad"][i]):
                p.grad.copy_(s["grads"][i])
            else:
                p.grad = None
        opt.step()
        for k, p in ps.items():
            s = rec["params"][k]
            assert _rel(p, s["ps"][i]) < 2e-6, (k, i)
            has = "momentum_buffer" in opt.state.get(p, {})
            assert has == bool(s["has_buf"][i]), (k, i)
            if has:
                assert _rel(opt.state[p]["momentum_buffer"], s["bufs"][i]) < 1e-5, (k, i)
    if tag == "dampening":    # b's first momentum step is step 4: buffer = g + wd*p, not (1-d)*that
        b = rec["params"]["b"]
        assert not bool(b["has_buf"][2]) and bool(b["has_buf"][3])


def test_sgd_multi_tensor_slimmable_ema_scale(built_lib):
    """Several tensors (odd sizes -> padded arena), the 'slimmable' mask folded in, EMA warm-up
    rule, 1/world gradient scale, nesterov, bf16 mirror — against tests/sgd_oracle.py."""
    from yet_another_mobilenet_series_b200.fused_sgd import SGD
    torch.manual_seed(0)
    shapes = {"features.0.0.weight": (8, 3, 3, 3), "features.0.1.weight": (8,),
              "features.0.1.bias": (8,), "features.1.ops.0.0.0.weight": (8, 1, 3, 3),
              "features.2.ops.1.2.weight": (8, 1, 1, 1), "features.2.ops.0.0.0.weight": (13, 8, 1, 1),
              "classifier.1.weight": (5, 13), "classifier.1.bias": (5,)}
    params = {k: torch.nn.Parameter(torch.randn(s).cuda()) for k, s in shapes.items()}
    kw = dict(lr=0.05, momentum=0.9, nesterov=True)
    opt = SGD(list(params.values()), **kw)
    opt.fold_l2(1e-2, list(params.items()), "slimmable")
    decay = 0.9999 ** (256 / 4096.0)
    opt.attach_ema(decay)
    opt.grad_scale = 0.25
    mask = so.l2_decay_mask(list(shapes.items()), "slimmable")
    assert not mask["features.2.ops.1.2.weight"] and mask["features.0.0.weight"]
    ref = {k: dict(p=v.detach().cpu().numpy().ravel().copy(), buf=None) for k, v in params.items()}
    for k in ref:
        ref[k]["ema"] = ref[k]["p"].copy()
    for t in range(1, 12):
        opt.zero_grad()
        for k, p in params.items():
            g = torch.randn(p.shape) * 2
            p.grad.copy_(g)
            r = ref[k]
            gg = g.numpy().ravel().astype(np.float32) * np.float32(0.25)
            if mask[k]:
                gg = gg + so.l2_grad(r["p"], 1e-2)
            r["p"], r["buf"] = so.sgd_step(r["p"], gg, r["buf"], **kw)
            r["ema"] = so.oo.ema_update(r["ema"], r["p"], decay, t)
        opt.step(num_updates=t)
    for k, p in params.items():
        assert _rel(p, ref[k]["p"].reshape(p.shape)) < 1e-5, k
        assert _rel(opt.state[p]["momentum_buffer"], ref[k]["buf"].reshape(p.shape)) < 1e-5, k
        assert _rel(opt.ema_shadow(p), ref[k]["ema"].reshape(p.shape)) < 1e-5, k
        assert torch.equal(p._yamb_bf16, p.detach().to(torch.bfloat16))
        assert p.grad.data_ptr() >= opt.arenas()["g"].data_ptr()


def _params(seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(s, generator=g).cuda()) for s in ((7, 5), (11,), (3,))]


def _run(opt, ps, grads):
    """Steps with the given gradients; the last parameter never has one."""
    for gs in grads:
        opt.zero_grad()
        for p, g in zip(ps[:-1], gs):
            if p.grad is None:
                p.grad = g.clone()
            else:
                p.grad.copy_(g)
        ps[-1].grad = None
        opt.step()


@pytest.mark.parametrize("src", ["fused", "torch"])
def test_state_dict_interchange_with_torch(built_lib, src):
    from yet_another_mobilenet_series_b200.fused_sgd import SGD
    kw = dict(lr=0.05, momentum=0.9, nesterov=True)
    torch.manual_seed(1)
    grads = [[torch.randn(7, 5, device="cuda"), torch.randn(11, device="cuda")] for _ in range(6)]
    a_cls, b_cls = (SGD, torch.optim.SGD) if src == "fused" else (torch.optim.SGD, SGD)
    pa = _params(0)
    oa = a_cls(pa, **kw)
    _run(oa, pa, grads[:3])
    sd = oa.state_dict()
    assert set(sd["state"]) == {0, 1}                 # the never-stepped parameter has no entry
    assert all(set(v) == {"momentum_buffer"} for v in sd["state"].values())
    pb = [torch.nn.Parameter(p.detach().clone()) for p in pa]
    ob = b_cls(pb, **kw)
    ob.load_state_dict(copy.deepcopy(sd))             # what torch.save / torch.load hand over
    assert ob.state_dict()["state"].keys() == {0, 1}
    _run(oa, pa, grads[3:])
    _run(ob, pb, grads[3:])
    for a, b in zip(pa, pb):
        assert _rel(b, a) < 2e-6
    for i in range(2):
        assert _rel(ob.state[pb[i]]["momentum_buffer"], oa.state[pa[i]]["momentum_buffer"]) < 1e-5
    assert torch.equal(pa[2], pb[2]) and pb[2] not in ob.state and pa[2] not in oa.state


def test_step_uses_grads_that_left_the_arena_and_skips_gradless_params(built_lib):
    """`model.zero_grad(set_to_none=True)` detaches the `.grad` views; autograd then allocates
    fresh gradient tensors.  step() must use them (copy into the arena, re-attach), and a
    parameter without a gradient is skipped like torch.optim.SGD does: no update, no buffer."""
    from yet_another_mobilenet_series_b200.fused_sgd import SGD
    torch.manual_seed(0)
    a = torch.nn.Parameter(torch.randn(37, device="cuda"))
    b = torch.nn.Parameter(torch.randn(5, 3, device="cuda"))
    opt = SGD([a, b], lr=0.1, momentum=0.9, nesterov=True)
    opt.arenas()
    a0, b0 = a.detach().clone(), b.detach().clone()
    a.grad = None
    b.grad = None                                   # what nn.Module.zero_grad() does
    (a * 2.0).sum().backward()                      # fresh .grad tensor for a, none for b
    assert a.grad.data_ptr() != opt.arenas()["gptr"][0]
    opt.step()
    torch.cuda.synchronize()
    want = a0 - 0.1 * (2.0 + 0.9 * 2.0)             # first step: buf = g; nesterov g + m*buf
    assert torch.allclose(a, want, rtol=1e-6, atol=1e-7)
    assert torch.equal(b, b0)                       # skipped: no state change at all
    assert "momentum_buffer" in opt.state[a] and b not in opt.state
    assert float(opt.arenas()["mom"][opt.arenas()["offs"][1]:].abs().max()) == 0.0
    assert a.grad.data_ptr() == opt.arenas()["gptr"][0]   # re-attached to the arena


def _flat(d, keys):
    return torch.cat([d[k].detach().double().flatten().cpu() for k in keys])


def _rel_t(a, b):
    return float((a - b).norm() / (b.norm() + 1e-30))


def _three_steps_vs_reference(name, B, ts_kw, ref_kw, l2_loss, ema):
    """test_configs_gpu.py's comparison: three TrainStep iterations against the reference step
    sequence in fp32 (truth) and autocast-bf16 (yardstick)."""
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda")
    model, cfg = build_from_cfg(name)
    for m in model.modules():          # dropout streams differ between the three runs: off
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    from oracle import torch_model as tm
    ref32 = so.RefTrainer(tm.as_reference(model).to(dev), B, **ref_kw)
    ref16 = so.RefTrainer(tm.as_reference(model).to(dev).to(memory_format=torch.channels_last), B,
                          autocast=torch.bfloat16, **ref_kw)
    p0 = {k: v.detach().clone() for k, v in model.named_parameters()}
    model = model.to(dev)
    ts = TrainStep(model, B, image_size=cfg["flags"]["image_size"], **ts_kw)
    wd = ts_kw["weight_decay"]
    g = torch.Generator().manual_seed(0)
    keys = [k for k, _ in model.named_parameters()]
    losses = {"ours": [], "fp32": [], "autocast": []}
    snaps = []
    for i in range(3):
        x = torch.randn(B, 3, 224, 224, generator=g).bfloat16()
        t = torch.randint(0, 1000, (B,), generator=g)
        xd, td = x.to(dev).float(), t.to(dev)
        l2 = float(l2_loss(ref32.model, wd))
        losses["fp32"].append(ref32.step(xd, td) - l2)           # TrainStep folds L2 into the update
        l2 = float(l2_loss(ref16.model, wd))
        losses["autocast"].append(ref16.step(xd.contiguous(memory_format=torch.channels_last), td) - l2)
        losses["ours"].append(float(ts(x, t)))
        snaps.append({k: v.detach().clone() for k, v in model.named_parameters()})
    torch.cuda.synchronize()
    assert ts.graph is not None                                   # the 3rd call replayed the graph
    rows = ["%s N=%d %s losses ours %s fp32 %s autocast %s" % (
        name, B, ts_kw.get("optimizer", "rmsprop"), losses["ours"], losses["fp32"],
        losses["autocast"])]
    try:
        for i in range(3):
            eo = abs(losses["ours"][i] - losses["fp32"][i])
            ea = abs(losses["autocast"][i] - losses["fp32"][i])
            assert eo <= 2.0 * ea + 5e-3 * abs(losses["fp32"][i]), rows
        pt = dict(ref32.model.named_parameters())
        pa = dict(ref16.model.named_parameters())
        po = dict(model.named_parameters())
        p0f = _flat(p0, keys)
        d_t, d_a, d_o = _flat(pt, keys) - p0f, _flat(pa, keys) - p0f, _flat(po, keys) - p0f
        eo, ea = _rel_t(d_o, d_t), _rel_t(d_a, d_t)
        rows.append("update rel-L2: ours %.4f autocast %.4f" % (eo, ea))
        assert eo <= 1.3 * ea + 1e-2, rows
        if ema:
            decay = ts_kw["ema_decay"] ** (B / ts_kw["ema_base_batch"])
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
            s_o = torch.cat([ts.opt.ema_shadow(po[k]).detach().double().flatten().cpu()
                             for k in keys]) - p0f
            assert _rel_t(s_o, s_t) <= 1.3 * _rel_t(s_a, s_t) + 1e-2, rows
        else:
            assert ts.ema_decay is None and ts.opt.arenas()["ema"] is None
        bt = dict(ref32.model.named_buffers())
        ba = dict(ref16.model.named_buffers())
        bo = dict(model.named_buffers())
        for kind in ("running_mean", "running_var"):
            ks = [k for k in bt if k.endswith(kind)]
            eo = sorted(_rel_t(bo[k].double().cpu(), bt[k].double().cpu()) for k in ks)
            ea = sorted(_rel_t(ba[k].double().cpu(), bt[k].double().cpu()) for k in ks)
            mo, ma = sum(eo) / len(eo), sum(ea) / len(ea)
            qo, qa = eo[int(0.9 * (len(eo) - 1))], ea[int(0.9 * (len(ea) - 1))]
            rows.append("%s per-buffer rel-L2: mean ours %.2e autocast %.2e; p90 ours %.2e "
                        "autocast %.2e" % (kind, mo, ma, qo, qa))
            assert mo <= 1.5 * ma + 2e-3, rows
            assert qo <= 1.5 * qa + 2e-3, rows
        nbt = [k for k in bt if k.endswith("num_batches_tracked")]
        assert all(int(bo[k]) == int(bt[k]) == 3 for k in nbt)
        if ema:
            sk = [n for n, b in model.named_buffers() if "running_mean" in n or "running_var" in n]
            eo = [_rel_t(s.detach().double().cpu(), ref32.ema.shadow[k].double().cpu())
                  for s, k in zip(ts.stat_shadow, sk)]
            ea = [_rel_t(ref16.ema.shadow[k].double().cpu(), ref32.ema.shadow[k].double().cpu())
                  for k in sk]
            mo, ma = sum(eo) / len(eo), sum(ea) / len(ea)
            rows.append("stat-shadow per-buffer mean rel-L2: ours %.2e autocast %.2e" % (mo, ma))
            assert mo <= 1.5 * ma + 2e-3, rows
    finally:
        print("\n".join(rows))


def _sgd_kw(ema_decay=EMA_DECAY, ema_base_batch=4096):
    common = dict(base_lr=BASE_LR, base_total_batch=BASE_TOTAL_BATCH, momentum=MOMENTUM,
                  weight_decay=WEIGHT_DECAY, label_smoothing=LABEL_SMOOTHING, ema_decay=ema_decay,
                  ema_base_batch=ema_base_batch)
    ts_kw = dict(common, optimizer="sgd", nesterov=NESTEROV, weight_decay_method="slimmable")
    ref_kw = dict(common, optimizer="sgd", nesterov=NESTEROV, weight_decay_method="slimmable")
    return ts_kw, ref_kw


@pytest.mark.parametrize("name,ema", [("mobilenet_v2", False), ("atomnas_c+", True)])
def test_trainstep_sgd_slimmable_vs_reference(built_lib, name, ema):
    if ema:       # the EMA of the model's own yml
        fl = load_cfgs()[name]["flags"]
        ts_kw, ref_kw = _sgd_kw(fl["moving_average_decay"], fl["moving_average_decay_base_batch"])
    else:
        ts_kw, ref_kw = _sgd_kw()
    _three_steps_vs_reference(name, 32, ts_kw, ref_kw, so.l2_loss_slimmable, ema)


def test_trainstep_rmsprop_slimmable_vs_reference(built_lib):
    name = "mobilenet_v2"
    fl = load_cfgs()[name]["flags"]
    common = dict(base_lr=fl["base_lr"], base_total_batch=fl["base_total_batch"], alpha=fl["alpha"],
                  momentum=fl["momentum"], eps=fl["epsilon"], weight_decay=fl["weight_decay"],
                  label_smoothing=fl["label_smoothing"], ema_decay=fl["moving_average_decay"],
                  ema_base_batch=fl["moving_average_decay_base_batch"])
    ts_kw = dict(common, weight_decay_method="slimmable")
    ref_kw = dict(common, weight_decay_method="slimmable")
    _three_steps_vs_reference(name, 32, ts_kw, ref_kw, so.l2_loss_slimmable, True)


ROWS = [[1, 16, 1, 1, [3]], [6, 24, 2, 2, [3]], [6, 32, 2, 2, [3]], [6, 64, 2, 2, [3]],
        [6, 96, 1, 1, [3]], [6, 160, 2, 2, [3]], [6, 320, 1, 1, [3]]]


def test_sgd_graph_replay_equals_eager(built_lib):
    """Two SGD iterations from the same state on the same batch, eagerly and as CUDA-graph
    replays: the same bits (the weight-gradient reductions add their partials in a fixed order,
    and the optimizer step is one deterministic kernel)."""
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb, mobilenet_supernet as sup
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    B = 32
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, 3, 96, 96, generator=g).to(torch.bfloat16)
    t = torch.randint(0, 100, (B,), generator=g)
    torch.manual_seed(1995)
    m = sup.Model(inverted_residual_setting=ROWS, active_fn="nn.ReLU", batch_norm_momentum=0.01,
                  batch_norm_epsilon=1e-3, num_classes=100, dropout_ratio=0.0, input_size=96)
    m.apply(mb.init_weights_mnas)
    m = m.cuda()
    ts_kw, _ = _sgd_kw()
    ts = TrainStep(m, B, image_size=96, **ts_kw)
    for _ in range(2):
        ts(x, t)                                  # two eager warm-up iterations
    torch.cuda.synchronize()
    A = ts.opt.arenas()
    st = {k: A[k].clone() for k in ("p", "mom", "bf16")}
    st["buf"] = {k: v.clone() for k, v in m.named_buffers()}

    def restore():
        with torch.no_grad():
            for k in ("p", "mom", "bf16"):
                A[k].copy_(st[k])
            for k, v in m.named_buffers():
                v.copy_(st["buf"][k])

    def two_steps():
        out = []
        for _ in range(2):
            loss = float(ts(x, t))
            out.append((loss, A["p"].clone(), A["mom"].clone()))
        return out

    ts.use_graph = False
    eager = two_steps()
    restore()
    ts.use_graph = True
    graph = two_steps()                           # captures, then replays
    torch.cuda.synchronize()
    assert ts.graph is not None
    for (le, pe, me), (lg, pg, mg) in zip(eager, graph):
        assert le == lg
        assert torch.equal(pe, pg) and torch.equal(me, mg)
    assert not torch.equal(eager[0][1], eager[1][1])   # the second step moved the weights
