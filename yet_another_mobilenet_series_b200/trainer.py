"""Public training-step API of the sm_90a path: `TrainStep(model, ...)(x, target)`.

One call = one iteration of the reference's hot loop (train.py:64-114): zero_grad, forward,
label-smoothed cross entropy (utils/optim.py:150-158) [+ top-k counts without the reference's two
host syncs, common.py:67-80], backward, gradient all-reduce (utils/distributed.py:155-161),
optimizer step with the L2 decay, the 1/world mean, the bf16 weight repack and the EMA of the
weights folded in, and the EMA of the BatchNorm running statistics (common.py:58-63).  The
optimizer is the reference's RMSprop (utils/rmsprop.py, the default) or torch.optim.SGD
(`optimizer="sgd"`, utils/optim.py:262-267), and the L2 rule `cal_l2_loss`'s 'mnas' (the default)
or 'slimmable' (utils/optim.py:161-200); EMA: utils/optim.py:53-64.

Forward+backward are captured once into a CUDA graph (static input buffers) and replayed; inputs
arrive through `load(x, target)` which accepts HOST (ideally pinned) or device tensors and copies
them on a side stream so the H2D copy of step i+1 overlaps the compute of step i (the role of the
reference's DataPrefetcher, utils/dataflow.py:13-58).
"""
import torch
import torch.distributed as dist

from . import distributed as udist
from . import engine
from . import tail_ops
from .fused_rmsprop import RMSprop
from .fused_sgd import SGD


def label_smooth_ce(logits, target, smoothing):
    """Per-sample label-smoothed CE (reference CrossEntropyLabelSmooth, reduction='none')."""
    logp = torch.log_softmax(logits.float(), 1)
    nll = -logp.gather(1, target.unsqueeze(1)).squeeze(1)
    return (1.0 - smoothing) * nll - (smoothing / logits.size(1)) * logp.sum(1)


class TrainStep:
    def __init__(self, model, per_gpu_batch, image_size=224, base_lr=0.016, base_total_batch=256,
                 alpha=0.9, momentum=0.9, eps=1e-3, weight_decay=1e-5, label_smoothing=0.1,
                 ema_decay=0.9999, ema_base_batch=4096, use_graph=True, input_dtype=torch.bfloat16,
                 optimizer="rmsprop", nesterov=False, dampening=0.0, weight_decay_method="mnas"):
        """`alpha` and `eps` apply to RMSprop only; `nesterov` and `dampening` to SGD only;
        `momentum`, `weight_decay` (folded in by `weight_decay_method`) and the EMA to both."""
        self.model = model
        dev = next(model.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("TrainStep needs the model on a CUDA device (no CPU path)")
        self.dev = dev
        self.world = udist.get_world_size_fallback()
        self.batch = per_gpu_batch
        gbatch = per_gpu_batch * self.world
        self.lr = base_lr * gbatch / base_total_batch            # reference common.py:204-205
        if optimizer == "rmsprop":
            self.opt = RMSprop(model.parameters(), lr=self.lr, alpha=alpha, momentum=momentum,
                               eps=eps, eps_inside_sqrt=True, weight_decay=0)
        elif optimizer == "sgd":                                  # utils/optim.py:262-267
            self.opt = SGD(model.parameters(), lr=self.lr, momentum=momentum,
                           dampening=dampening, nesterov=nesterov, weight_decay=0)
        else:
            raise ValueError("Unknown optimizer: {}".format(optimizer))
        self.opt.fold_l2(weight_decay, list(model.named_parameters()), weight_decay_method)
        self.ema_decay = None
        if ema_decay and ema_decay > 0:
            self.ema_decay = ema_decay ** (gbatch / ema_base_batch)  # adjust_momentum, :118-128
            self.opt.attach_ema(self.ema_decay)
        self.opt.grad_scale = 1.0 / self.world
        self.opt.arenas()
        self.smoothing = label_smoothing
        # BN running statistics and their EMA shadows (flat, for one fused update)
        self.stat_bufs = [b for n, b in model.named_buffers()
                          if "running_mean" in n or "running_var" in n]
        self.stat_shadow = [b.detach().clone() for b in self.stat_bufs]
        # static buffers
        self.x = torch.zeros(per_gpu_batch, 3, image_size, image_size, device=dev,
                             dtype=input_dtype).contiguous(memory_format=torch.channels_last)
        self.t = torch.zeros(per_gpu_batch, dtype=torch.long, device=dev)
        # staging copies: the H2D transfer of batch i+1 lands here while the graph of step i still
        # reads self.x / self.t; a device-to-device move at the start of step i+1 publishes it
        self.x_stage = torch.zeros_like(self.x)
        self.t_stage = torch.zeros_like(self.t)
        self.staged = False
        self.loss = torch.zeros((), device=dev)
        self.top1 = torch.zeros((), device=dev)   # fraction correct@1 / @5 of the last batch
        self.top5 = torch.zeros((), device=dev)
        self.copy_stream = torch.cuda.Stream(device=dev)
        self.copied = torch.cuda.Event()
        self.consumed = torch.cuda.Event()
        self.consumed.record()
        self.use_graph = use_graph
        self.graph = None
        self.global_step = 0
        self.launches_per_step = None
        self._warm = 0

    # ---- input path ----------------------------------------------------------------------------
    def load(self, x, target):
        """Stage the next batch into the static device buffers (async on the copy stream)."""
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self.consumed)  # staging buffers were drained
            self.x_stage.copy_(x, non_blocking=True)
            self.t_stage.copy_(target, non_blocking=True)
            self.copied.record(self.copy_stream)
        self.staged = True

    # ---- one iteration -------------------------------------------------------------------------
    def _fwd_bwd(self):
        self.opt.zero_grad()
        logits = self.model(self.x)
        # label-smoothed CE + top-1 / top-5 in one kernel, no host sync (common.py:67-80)
        per_sample, c1, c5 = tail_ops.softmax_ce(logits, self.t, self.smoothing)
        loss = per_sample.mean()
        engine.DEFER_JOIN = True      # wgrad side stream: one join after the whole backward
        try:
            loss.backward()
        finally:
            engine.DEFER_JOIN = False
            engine.join_side(self.dev)
        self.loss.copy_(loss.detach())
        self.top1.copy_(c1.mean())
        self.top5.copy_(c5.mean())

    def _capture(self):
        g = torch.cuda.CUDAGraph()
        before = engine.LAUNCHES
        with torch.cuda.graph(g):
            self._fwd_bwd()
        self.launches_per_step = engine.LAUNCHES - before + 1  # + fused optimizer kernel
        self.graph = g

    def run(self):
        """Run one iteration on the staged batch; returns the (device) loss tensor."""
        cur = torch.cuda.current_stream()
        if self.staged:
            cur.wait_event(self.copied)
            self.x.copy_(self.x_stage)
            self.t.copy_(self.t_stage)
            self.consumed.record(cur)
            self.staged = False
        self.model.train()
        self.opt.sync_mirror()   # masters written in place since the last step (load_state_dict ...)
        if self.use_graph and self.graph is None and self._warm >= 2:
            torch.cuda.synchronize()
            self._capture()
        if self.graph is not None:
            self.graph.replay()
        else:
            before = engine.LAUNCHES
            self._fwd_bwd()
            self.launches_per_step = engine.LAUNCHES - before + 1
            self._warm += 1
        if self.world > 1:
            dist.all_reduce(self.opt.arenas()["g"])   # in place on the flat arena; mean is folded
        self.global_step += 1
        self.opt.step(num_updates=self.global_step)
        if self.ema_decay is not None and self.stat_bufs:
            m = self.opt.ema_momentum(self.global_step)
            torch._foreach_mul_(self.stat_shadow, m)
            torch._foreach_add_(self.stat_shadow, self.stat_bufs, alpha=1.0 - m)
        return self.loss

    def __call__(self, x, target):
        self.load(x, target)
        return self.run()
