"""GPU: the whole MobileNetV2 through the sm_90a path vs the plain-torch port of the reference
graph (oracle/torch_model.py, fp32 on CPU), and TrainStep (CUDA graph, flat-arena optimizer)
vs the reference step sequence."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

ROWS = [[1, 16, 1, 1, [3]], [6, 24, 2, 2, [3]], [6, 32, 2, 2, [3]], [6, 64, 2, 2, [3]],
        [6, 96, 1, 1, [3]], [6, 160, 2, 2, [3]], [6, 320, 1, 1, [3]]]
KW = dict(inverted_residual_setting=ROWS, active_fn="nn.ReLU", batch_norm_momentum=0.01,
          batch_norm_epsilon=1e-3, num_classes=100, dropout_ratio=0.0)


def _rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-20))


def _model(input_size):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb, mobilenet_supernet as sup
    torch.manual_seed(1995)
    m = sup.Model(**KW, input_size=input_size)
    m.apply(mb.init_weights_mnas)
    return m


def test_eval_logits_match_reference_graph(built_lib):
    from oracle import torch_model as tm
    m = _model(96)
    g = torch.Generator().manual_seed(3)
    for mod in m.modules():  # non-trivial running statistics
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.running_mean.normal_(0, 0.1, generator=g)
            mod.running_var.uniform_(0.7, 1.3, generator=g)
    ref = tm.as_reference(m).eval()
    x = torch.randn(8, 3, 96, 96, generator=g)
    with torch.no_grad():
        want = ref(x)
        got = m.cuda().eval()(x.cuda())
    assert got.dtype == torch.float32 and got.shape == want.shape
    assert _rel(got, want) < 3e-2  # 17 bf16 blocks deep; reference autocast-bf16 is ~5e-3/block


def test_train_step_matches_reference_sequence(built_lib):
    """4 iterations of TrainStep (graph replay from the 3rd) vs oracle RefTrainer on CPU fp32 with
    the same data on a toy size: first loss, the EMA recurrence (exact) and "it trains".  The
    trajectory parity at the real configurations, with the autocast yardstick, lives in
    tests/test_configs_gpu.py."""
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    B = 16
    m = _model(64)
    ref = tm.as_reference(m)
    trainer = tm.RefTrainer(ref, B)
    w0 = m.classifier[1].weight.detach().clone()
    m = m.cuda()
    ts = TrainStep(m, B, image_size=64)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, 3, 64, 64, generator=g)
    t = torch.randint(0, 100, (B,), generator=g)
    losses_ref, losses, snaps = [], [], []
    for i in range(4):
        l2 = float(tm.l2_loss_mnas(ref, 1e-5))
        losses_ref.append(trainer.step(x, t) - l2)  # TrainStep folds L2 into the update
        losses.append(float(ts(x.to(torch.bfloat16), t)))
        snaps.append(m.classifier[1].weight.detach().clone())
    torch.cuda.synchronize()
    assert ts.graph is not None
    assert abs(losses[0] - losses_ref[0]) < 2e-2 * abs(losses_ref[0])
    assert losses[-1] < 0.5 * losses[0] and losses_ref[-1] < 0.5 * losses_ref[0]  # both train
    # EMA shadow of a weight: the recurrence of utils/optim.py:56-64 on OUR weight trajectory,
    # m = min(decay_adjusted, (1 + t) / (10 + t)) with t the incremented global step (train.py:109)
    decay = 0.9999 ** (B / 4096)
    sh = w0.cuda()
    for step, w in enumerate(snaps, 1):
        mm = min(decay, (1.0 + step) / (10.0 + step))
        sh = mm * sh + (1.0 - mm) * w
    got = ts.opt.ema_shadow(m.classifier[1].weight)
    assert float((got - sh).abs().max()) < 1e-6 * float(sh.abs().max()) + 1e-9
    # ... and it is what the reference's EMA holds for ITS trajectory, within the bf16 budget
    ref_sh = trainer.ema.shadow["classifier.1.weight"]
    assert _rel(got - w0.cuda(), ref_sh - w0) < 0.4   # toy size; real sizes: test_configs_gpu.py


def test_first_step_gradients_match_reference_graph(built_lib):
    """Whole-network gradients of one forward/backward (flat-arena direct accumulation mode).

    Truth = autograd of the fp32 reference graph on CPU.  The yardstick is the reference's OWN
    bf16 path (the same stock-torch graph under torch.autocast(bfloat16) on the GPU, SURVEY.md
    §8c gate ii): this path must be as close to the fp32 truth as that one, layer by layer.
    (BatchNorm-gamma gradients of layers whose beta is 0 are structurally ~0 — the following
    BatchNorm removes the scale — so only >=2-D weights are compared.)"""
    from oracle import torch_model as tm
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    B = 32
    m = _model(64)
    ref = tm.as_reference(m).train()
    ref16 = tm.as_reference(m).cuda().train()
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, 3, 64, 64, generator=g)
    t = torch.randint(0, 100, (B,), generator=g)
    tm.label_smooth_ce(ref(x), t, 0.1).mean().backward()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out16 = ref16(x.cuda().to(memory_format=torch.channels_last))
    tm.label_smooth_ce(out16.float(), t.cuda(), 0.1).mean().backward()
    m = m.cuda()
    ts = TrainStep(m, B, image_size=64, use_graph=False)
    ts.load(x.to(torch.bfloat16), t)
    ts.x.copy_(ts.x_stage)
    ts.t.copy_(ts.t_stage)
    m.train()
    ts._fwd_bwd()
    torch.cuda.synchronize()
    refp, ref16p = dict(ref.named_parameters()), dict(ref16.named_parameters())

    def cos(a, b):
        a, b = a.detach().float().cpu().flatten(), b.detach().float().cpu().flatten()
        return float(torch.dot(a, b) / (a.norm() * b.norm() + 1e-30))

    ours, auto, report = [], [], []
    for k, p in m.named_parameters():
        if p.dim() < 2:
            continue
        co, ca = cos(p.grad, refp[k].grad), cos(ref16p[k].grad, refp[k].grad)
        ours.append(co)
        auto.append(ca)
        report.append("%-36s ours=%.4f torch-autocast=%.4f" % (k, co, ca))
    print("\n".join(report))
    mo, ma = sum(ours) / len(ours), sum(auto) / len(auto)
    print("mean cosine to fp32 truth: ours %.4f, torch autocast-bf16 %.4f" % (mo, ma))
    assert mo > ma - 0.03, (mo, ma)
    assert min(o - a for o, a in zip(ours, auto)) > -0.12, report


def _state(ts, model):
    A = ts.opt.arenas()
    st = {k: A[k].clone() for k in ("p", "sq", "mom", "ema", "bf16") if A.get(k) is not None}
    st["buf"] = {k: v.clone() for k, v in model.named_buffers()}
    st["shadow"] = [s.clone() for s in ts.stat_shadow]
    st["step"] = ts.global_step
    return st


def _restore(ts, model, st):
    A = ts.opt.arenas()
    with torch.no_grad():
        for k in ("p", "sq", "mom", "ema", "bf16"):
            if k in st:
                A[k].copy_(st[k])
        for k, v in model.named_buffers():
            v.copy_(st["buf"][k])
        for s, v in zip(ts.stat_shadow, st["shadow"]):
            s.copy_(v)
    ts.global_step = st["step"]


def test_graph_replay_equals_eager(built_lib):
    """The SAME iteration (same state, same batch) run eagerly TWICE and once as a CUDA-graph
    replay.  Everything that crosses warps or CTAs in the BatchNorm statistics is accumulated in
    double (csrc/bn_finalize.cuh), so the forward pass and every activation gradient are the same
    bits run after run; the weight-gradient reductions (split-K GEMM, depthwise, stem, classifier
    bias) add per-CTA partials in a fixed order (csrc/det_reduce.cu).  (With fp32 statistics
    atomics, round 1, two eager runs differed by 1.6e-3 in the loss and 0.2 in the update: bf16
    rounding flips amplified the last-bit differences of the BatchNorm coefficients.)"""
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    B = 32
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, 3, 96, 96, generator=g).to(torch.bfloat16)
    t = torch.randint(0, 100, (B,), generator=g)
    m = _model(96).cuda()
    for mod in m.modules():  # the dropout stream differs between capture and eager: switch it off
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    ts = TrainStep(m, B, image_size=96)
    for _ in range(2):
        ts(x, t)                                  # two eager warm-up iterations
    torch.cuda.synchronize()
    st = _state(ts, m)
    ts.use_graph = False
    loss_e = float(ts(x, t))
    p_e = ts.opt.arenas()["p"].clone()
    _restore(ts, m, st)
    loss_e2 = float(ts(x, t))                     # eager twice: the reduction-order noise itself
    p_e2 = ts.opt.arenas()["p"].clone()
    _restore(ts, m, st)
    ts.use_graph = True
    loss_g = float(ts(x, t))                      # captures, then replays
    torch.cuda.synchronize()
    assert ts.graph is not None
    p_g = ts.opt.arenas()["p"].clone()
    noise = _rel(p_e2 - st["p"], p_e - st["p"])
    diff = _rel(p_g - st["p"], p_e - st["p"])
    print("eager-vs-eager update rel-L2 %.3e, graph-vs-eager %.3e; losses %r %r %r"
          % (noise, diff, loss_e, loss_e2, loss_g))
    assert abs(loss_e2 - loss_e) <= 1e-6 * abs(loss_e)
    assert abs(loss_g - loss_e) <= 1e-6 * abs(loss_e)
    assert noise < 1e-4 and diff < 1e-4
    # the weight-gradient reductions add their partials in a fixed order: the same bits every time
    assert torch.equal(p_e2, p_e) and torch.equal(p_g, p_e)
    # a larger eager step in between (bigger reduction scratch) must not disturb the captured graph
    big = _model(128).cuda()
    ts_big = TrainStep(big, 2 * B, image_size=128, use_graph=False)
    xb = torch.randn(2 * B, 3, 128, 128, generator=g).to(torch.bfloat16)
    ts_big(xb, torch.randint(0, 100, (2 * B,), generator=g))
    torch.cuda.synchronize()
    _restore(ts, m, st)
    assert float(ts(x, t)) == loss_g              # replay of the graph captured above
    assert torch.equal(ts.opt.arenas()["p"], p_g)
    # replaying again advances the training (the graph is not a frozen snapshot)
    loss_next = float(ts(x, t))
    assert loss_next < loss_g
