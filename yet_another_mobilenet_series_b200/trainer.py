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
reference's DataPrefetcher, utils/dataflow.py:13-58).  A batch of another shape (the partial last
batch of a `drop_last=False` loader, utils/dataflow.py:217-225) runs the same kernels eagerly and
leaves the graph in place.  The graph is captured again when the optimizer rebuilt the arenas it
holds pointers into.

Checkpoints have the layout of the reference's save_status (utils/common.py:122-133):
`state_dict` / `save_status` write it, `load_state_dict` continues from it (or from one the
reference wrote) by copying into the existing tensors; resuming is bit-exact.

The other half of an epoch, the reference's `validate()` (train.py:273-309), is
`TrainStep.validate`: `ema_model()` (get_ema_model, common.py:155-172) -> `EvalStep.calibrate`
(bn_calibration, utils/common.py:175-187) -> `EvalStep.evaluate` (forward_loss, common.py:67-80,
with the metrics summed on the device).

Both steps take uint8 image batches (`input_dtype=torch.uint8, input_norm=(mean, std)`, e.g. from
`dataflow.fast_collate`): the static buffers are then uint8 channels_last, `load` is a plain H2D
copy of a quarter of the fp32 bytes, and the stem kernels apply ToTensor() + Normalize(mean, std).

Gradient accumulation (`micro_batch`): one step runs k = per_gpu_batch / micro_batch forward and
backward passes over consecutive row slices of the batch into the one gradient arena, then one
all-reduce, one optimizer step and one EMA update, so a recipe's global batch (the reference's
`per_gpu_batch_size` x world) is reached with fewer GPUs: the global batch of a step is
per_gpu_batch x world, and the learning rate and EMA decay follow it.
"""
import copy
import os
from collections import OrderedDict

import torch
import torch.distributed as dist

from . import dataflow
from . import distributed as udist
from . import engine
from . import tail_ops
from .flat_arena import ema_momentum
from .fused_rmsprop import RMSprop
from .fused_sgd import SGD


def label_smooth_ce(logits, target, smoothing):
    """Per-sample label-smoothed CE (reference CrossEntropyLabelSmooth, reduction='none')."""
    logp = torch.log_softmax(logits.float(), 1)
    nll = -logp.gather(1, target.unsqueeze(1)).squeeze(1)
    return (1.0 - smoothing) * nll - (smoothing / logits.size(1)) * logp.sum(1)


def step_hyper(per_gpu_batch, micro_batch, world, base_lr=0.016, base_total_batch=256,
               ema_decay=0.9999, ema_base_batch=4096):
    """What a step of `per_gpu_batch` images per GPU, run in micro-batches of `micro_batch`
    (None: the whole batch) on `world` GPUs, derives: (micro_batch, k micro-batches per step,
    learning rate, EMA decay or None, optimizer grad_scale).  The learning rate and the EMA decay
    follow the global batch per_gpu_batch x world (reference common.py:47-57, 204-205); every
    micro-batch backpropagates its own mean loss, so grad_scale = 1 / (world x k) turns the sum
    over ranks and micro-batches into the mean over the global batch."""
    micro_batch = per_gpu_batch if micro_batch is None else micro_batch
    if micro_batch <= 0 or per_gpu_batch % micro_batch:
        raise ValueError("micro_batch must be a positive divisor of per_gpu_batch (got %r for %r)"
                         % (micro_batch, per_gpu_batch))
    k = per_gpu_batch // micro_batch
    gbatch = per_gpu_batch * world
    lr = base_lr * gbatch / base_total_batch                     # reference common.py:204-205
    decay = None
    if ema_decay and ema_decay > 0:
        decay = ema_decay ** (gbatch / ema_base_batch)           # adjust_momentum, :118-128
    return micro_batch, k, lr, decay, 1.0 / (world * k)


class TrainStep:
    def __init__(self, model, per_gpu_batch, image_size=224, base_lr=0.016, base_total_batch=256,
                 alpha=0.9, momentum=0.9, eps=1e-3, weight_decay=1e-5, label_smoothing=0.1,
                 ema_decay=0.9999, ema_base_batch=4096, use_graph=True, input_dtype=torch.bfloat16,
                 optimizer="rmsprop", nesterov=False, dampening=0.0, weight_decay_method="mnas",
                 input_norm=None, micro_batch=None, fused_tail=False, fused_stem=False,
                 fused_multi_branch=False, fused_se=False, fused_expand_dw=False,
                 grouped_branches=False):
        """`alpha` and `eps` apply to RMSprop only; `nesterov` and `dampening` to SGD only;
        `momentum`, `weight_decay` (folded in by `weight_decay_method`) and the EMA to both.
        `input_norm` = (mean, std) of the uint8 batches of `input_dtype=torch.uint8` (required
        there); it is attached to the model (dataflow.set_input_norm).

        `per_gpu_batch` is the number of images per GPU per optimizer step: the batch `load` and
        `__call__` take, and the batch the learning rate and the EMA decay are derived from.
        `micro_batch` (default `per_gpu_batch`, a divisor of it) is the number of images per
        forward and backward pass: a step accumulates the gradients of k = per_gpu_batch /
        micro_batch passes, captured together in one CUDA graph.  BatchNorm then behaves like the
        reference's per-GPU local BatchNorm at per_gpu_batch_size = micro_batch: batch statistics
        are those of each micro-batch, the running statistics are updated once per micro-batch (k
        times per step), and their EMA shadow once per step.  `micro_batch` is not part of a
        checkpoint: one written with any k loads into a TrainStep with any other.

        `fused_tail=True` runs the head BatchNorm + activation and the global average pool of this
        step's forwards and backwards as one kernel each way (engine.TRAIN_TAIL_FUSED): the
        activation and its broadcast gradient stay out of HBM.  Off by default: the pool sums in
        its own fixed order, not torch's, so a step with it differs from the default in the last
        bits.  A plain `model(x)` outside the step is not affected.

        `fused_stem=True` runs the stem ConvBNReLU of this step's forwards and backwards together
        with the first block when that block is the stem activation's only consumer (no
        expansion, no skip connection; engine.TRAIN_STEM_FUSED): the stem convolution takes the
        BatchNorm statistics, the block's depthwise applies the BatchNorm + activation on load
        and returns their backward, and the stem weight gradient forms dh on load, so the stem's
        activation, its gradient and dh stay out of HBM.  Off by default: the statistics are
        summed in another order (and with Swish dz is rounded after the act' product), so a step
        with it differs from the default in the last bits, the same bits on every run.  It
        combines with `fused_tail`; a plain `model(x)` outside the step is not affected.

        `fused_se=True` runs the Squeeze-and-Excitation backward of this step's blocks without a
        pass over the hidden tensor (engine.TRAIN_SE_FUSED): one reduction takes dgate and the
        per-(sample, channel) factors of BatchNorm-2's backward statistics, and the depthwise
        backward forms dz2 from dY, the gate and dpool while it stages its tiles, so dz2 is never
        written.  Off by default: BatchNorm-2's backward statistics are summed in another order, so
        a step with it differs from the default in the last bits, the same bits on every run.  It
        combines with `fused_stem` and `fused_tail`; a plain `model(x)` is not affected.

        `fused_expand_dw=True` runs the depthwise forward of this step's single-branch blocks with
        an expansion from x instead of reading h1 back (engine.TRAIN_EXPAND_DW_FUSED): each tile
        recomputes its expanded input with the expand GEMM's bf16 weights and BatchNorm-1
        coefficients, where engine.EXPAND_DW_SHAPE_RULE accepts the block's shape.  h2 has the
        default's bits; BatchNorm-2's statistics are summed in another order, so a step with it can
        differ from the default in the last bits.  It combines with `fused_stem`, `fused_tail`,
        `fused_se` and `micro_batch`; a plain `model(x)` is not affected.

        `grouped_branches=True` runs the depthwise of every branch of this step's multi-branch
        blocks with an expansion (AtomNAS, the single-path supernet) as one launch each way
        (engine.TRAIN_MB_DW_GROUPED) instead of one launch per branch: the grouped grid is the
        concatenation of the per-branch grids and each CTA runs what its per-branch CTA runs, so a
        step with it has the default's bits.  Only block kinds engine.MB_DW_SHAPE_RULE accepts are
        grouped; none by default, because grouping measured slower on an H100 (BASELINE.md §5).
        The backward of a block with Squeeze-and-Excitation
        keeps its per-branch launches under `fused_se`.  It is not recorded in checkpoints, and it
        combines with `micro_batch`, partial batches, `fused_stem`, `fused_tail`, `fused_se` and
        `fused_expand_dw`; a plain `model(x)` is not affected.

        `fused_multi_branch=True` is handed to the EvalStep that `validate` builds (see there)."""
        self.world = udist.get_world_size_fallback()
        self.micro_batch, self.accum, self.lr, self.ema_decay, self.grad_scale = step_hyper(
            per_gpu_batch, micro_batch, self.world, base_lr, base_total_batch, ema_decay,
            ema_base_batch)
        _attach_input_norm(model, input_dtype, input_norm)
        self.model = model
        dev = next(model.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("TrainStep needs the model on a CUDA device (no CPU path)")
        self.dev = dev
        self.batch = per_gpu_batch
        self.fused_tail = bool(fused_tail)
        self.fused_stem = bool(fused_stem)
        self.fused_se = bool(fused_se)
        self.fused_expand_dw = bool(fused_expand_dw)
        self.grouped_branches = bool(grouped_branches)
        self.fused_multi_branch = bool(fused_multi_branch)
        if optimizer == "rmsprop":
            self.opt = RMSprop(model.parameters(), lr=self.lr, alpha=alpha, momentum=momentum,
                               eps=eps, eps_inside_sqrt=True, weight_decay=0)
        elif optimizer == "sgd":                                  # utils/optim.py:262-267
            self.opt = SGD(model.parameters(), lr=self.lr, momentum=momentum,
                           dampening=dampening, nesterov=nesterov, weight_decay=0)
        else:
            raise ValueError("Unknown optimizer: {}".format(optimizer))
        self.opt.fold_l2(weight_decay, list(model.named_parameters()), weight_decay_method)
        if self.ema_decay is not None:
            self.opt.attach_ema(self.ema_decay)
        self.opt.grad_scale = self.grad_scale
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
        self.partial = None       # (x, target) of a batch of another shape, run eagerly
        self.loss = torch.zeros((), device=dev)
        self.top1 = torch.zeros((), device=dev)   # fraction correct@1 / @5 of the last batch
        self.top5 = torch.zeros((), device=dev)
        self.copy_stream = torch.cuda.Stream(device=dev)
        self.copied = torch.cuda.Event()
        self.consumed = torch.cuda.Event()
        self.consumed.record()
        self.use_graph = use_graph
        self.graph = None
        self._graph_arenas = None  # the optimizer arenas the graph holds raw pointers into
        self.global_step = 0
        self.launches_per_step = None
        self._warm = 0
        self._ema_model = None
        self._eval_step = None

    # ---- input path ----------------------------------------------------------------------------
    def load(self, x, target):
        """Stage the next batch into the static device buffers (async on the copy stream).  A batch
        of another shape (the partial last batch of a `drop_last=False` loader) is kept as given:
        `run` moves it to the device and runs that step eagerly."""
        if tuple(x.shape) != tuple(self.x.shape):
            self.partial = (x, target)
            return
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self.consumed)  # staging buffers were drained
            self.x_stage.copy_(x, non_blocking=True)
            self.t_stage.copy_(target, non_blocking=True)
            self.copied.record(self.copy_stream)
        self.staged = True

    # ---- one iteration -------------------------------------------------------------------------
    def _fwd_bwd(self, x=None, t=None):
        """Forward + loss + backward on (x, t), by default the static buffers, in passes of at
        most `micro_batch` rows whose gradients accumulate in the flat arena.  A batch of
        `per_gpu_batch` rows backpropagates the mean loss of every pass (grad_scale divides by
        their number k); any other batch of n rows (a partial last batch) weights the mean of a
        pass of n_i rows by n_i / n, a device scalar, so its gradient is that of the mean over the
        n rows."""
        engine.TRAIN_TAIL_FUSED = self.fused_tail
        engine.TRAIN_STEM_FUSED = self.fused_stem
        engine.TRAIN_SE_FUSED = self.fused_se
        engine.TRAIN_EXPAND_DW_FUSED = self.fused_expand_dw
        engine.TRAIN_MB_DW_GROUPED = self.grouped_branches
        try:
            self._passes(self.x if x is None else x, self.t if t is None else t)
        finally:
            engine.TRAIN_TAIL_FUSED = False
            engine.TRAIN_STEM_FUSED = False
            engine.TRAIN_SE_FUSED = False
            engine.TRAIN_EXPAND_DW_FUSED = False
            engine.TRAIN_MB_DW_GROUPED = False

    def _passes(self, x, t):
        n, b = x.shape[0], self.micro_batch
        self.opt.zero_grad()
        if n <= b:
            loss, _, c1, c5 = self._micro_step(x, t)
            self.loss.copy_(loss.detach())
            self.top1.copy_(c1.mean())
            self.top5.copy_(c5.mean())
            return
        weights = None
        if n != self.batch:
            weights = torch.tensor([min(b, n - s) / n for s in range(0, n, b)], device=self.dev)
        self.loss.zero_()
        self.top1.zero_()
        self.top5.zero_()
        for i, s in enumerate(range(0, n, b)):
            # a row slice of a channels_last batch is a channels_last view: no copy
            _, per_sample, c1, c5 = self._micro_step(x[s:s + b], t[s:s + b],
                                                     None if weights is None else weights[i])
            self.loss.add_(per_sample.detach().sum())
            self.top1.add_(c1.sum())
            self.top5.add_(c5.sum())
        self.loss.div_(n)
        self.top1.div_(n)
        self.top5.div_(n)

    def _micro_step(self, x, t, weight=None):
        """Forward, loss and backward of one pass; returns (the loss it backpropagated, the
        per-sample loss, correct@1, correct@5)."""
        logits = self.model(x)
        # label-smoothed CE + top-1 / top-5 in one kernel, no host sync (common.py:67-80)
        per_sample, c1, c5 = tail_ops.softmax_ce(logits, t, self.smoothing)
        loss = per_sample.mean()
        if weight is not None:
            loss = loss * weight
        engine.DEFER_JOIN = True      # wgrad side stream: one join after this pass's backward
        try:
            loss.backward()
        finally:
            engine.DEFER_JOIN = False
            # the side-stream weight-gradient GEMMs read block intermediates (h1, h2, dh3, the
            # BatchNorm coefficients) that the next pass's forward rewrites: join before it
            engine.join_side(self.dev)
        return loss, per_sample, c1, c5

    def _capture(self):
        g = torch.cuda.CUDAGraph()
        before = engine.LAUNCHES
        with torch.cuda.graph(g):
            self._fwd_bwd()
        self.launches_per_step = engine.LAUNCHES - before + 1  # + fused optimizer kernel
        self.graph = g
        self._graph_arenas = self.opt.arenas()

    def run(self):
        """Run one iteration on the staged batch; returns the (device) loss tensor."""
        cur = torch.cuda.current_stream()
        partial, self.partial = self.partial, None
        if partial is not None:
            x = torch.empty(partial[0].shape, device=self.dev, dtype=self.x.dtype,
                            memory_format=torch.channels_last)
            x.copy_(partial[0], non_blocking=True)
            t = partial[1].to(self.dev, dtype=self.t.dtype, non_blocking=True)
        elif self.staged:
            cur.wait_event(self.copied)
            self.x.copy_(self.x_stage)
            self.t.copy_(self.t_stage)
            self.consumed.record(cur)
            self.staged = False
        self.model.train()
        if self.graph is not None and self._graph_arenas is not self.opt.arenas():
            # the optimizer rebuilt its arenas (its load_state_dict, fold_l2, attach_ema): the
            # graph would accumulate into the freed gradient arena and read the old bf16 mirror
            self.graph = self._graph_arenas = None
            self._warm = 0
        self.opt.sync_mirror()   # masters written in place since the last step (load_state_dict ...)
        if partial is not None:
            self._fwd_bwd(x, t)   # eager; the graph and its pinned plans stay for full batches
        else:
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
        # a partial batch's passes are weighted to its mean already: only the ranks' sum is left
        self.opt.grad_scale = self.grad_scale if partial is None else 1.0 / self.world
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

    # ---- checkpoints ---------------------------------------------------------------------------
    def state_dict(self, epoch=None, best_val=None, meters=None):
        """The checkpoint of the reference's save_status (utils/common.py:122-133): 'model' (keys
        prefixed 'module.', as its DataParallel wrapper writes them), 'optimizer', 'ema' (the
        layout of its ExponentialMovingAverage.state_dict(), None without EMA), 'last_epoch',
        'best_val', 'meters'; plus 'global_step' and 'cuda_rng_state' (the model device's
        generator, for Dropout), which the reference ignores.  Tensors are the live ones, not
        copies."""
        ema = None
        if self.ema_decay is not None:
            pnames, snames = ema_names(self.model)
            shadow = OrderedDict((n, self.opt.ema_shadow(p))
                                 for n, p in zip(pnames, self.model.parameters()))
            shadow.update(zip(snames, self.stat_shadow))
            ema = ema_state_dict(shadow, self.global_step, self.ema_decay)
        return {"model": OrderedDict(("module." + k, v) for k, v in self.model.state_dict().items()),
                "optimizer": self.opt.state_dict(), "ema": ema, "last_epoch": epoch,
                "best_val": best_val, "meters": meters, "global_step": self.global_step,
                "cuda_rng_state": torch.cuda.get_rng_state(self.dev)}

    def save_status(self, path, epoch, best_val, meters):
        """`torch.save(self.state_dict(...), path)` on the master rank only (the reference's
        save_status).  The file is written next to `path` and renamed over it, so a run stopped
        while writing leaves the previous checkpoint intact."""
        sd = self.state_dict(epoch, best_val, meters)
        if udist.is_master():
            tmp = path + ".tmp"
            torch.save(sd, tmp)
            os.replace(tmp, path)

    def load_state_dict(self, ckpt):
        """Continue from a checkpoint of `state_dict` / `save_status`, or one the reference's
        save_status wrote: model (keys with or without 'module.'), optimizer state and
        hyper-parameters, EMA shadows of the weights and of the running statistics, `global_step`
        ('global_step', else the EMA's num_updates) and the CUDA generator state.  'optimizer' and
        'ema' may be absent or None; without 'ema' the EMA restarts from the loaded model.

        Everything is copied into the tensors that exist (the model's parameters are views of the
        optimizer's arenas), so a captured step graph stays valid and is replayed next."""
        model = OrderedDict((k[len("module."):] if k.startswith("module.") else k, v)
                            for k, v in ckpt["model"].items())
        self.model.load_state_dict(model)
        ema = ckpt.get("ema")
        shadows = None
        if self.ema_decay is not None:
            pnames, snames = ema_names(self.model)
            if ema is not None:
                shadows = [ema["shadow"][n] for n in pnames]
                stats = [ema["shadow"][n] for n in snames]
            else:
                shadows = list(self.model.parameters())
                stats = self.stat_bufs
            with torch.no_grad():
                for s, v in zip(self.stat_shadow, stats):
                    s.copy_(v)
        if ckpt.get("optimizer") is not None:
            self.opt.load_in_place(ckpt["optimizer"], ema=shadows)
        elif shadows is not None:
            with torch.no_grad():
                for p, s in zip(self.model.parameters(), shadows):
                    self.opt.ema_shadow(p).copy_(s)
        if ckpt.get("global_step") is not None:
            self.global_step = int(ckpt["global_step"])
        elif ema is not None and ema["info"]:
            self.global_step = int(next(iter(ema["info"].values()))["num_updates"])
        if ckpt.get("cuda_rng_state") is not None:
            torch.cuda.set_rng_state(ckpt["cuda_rng_state"].cpu(), self.dev)

    # ---- validation ----------------------------------------------------------------------------
    def ema_model(self):
        """The model with the EMA weights and EMA running statistics (reference get_ema_model,
        common.py:155-172).  Built once by `copy.deepcopy` (kernel scratch does not travel, and a
        copied Parameter has no `_yamb_bf16`, so the copy never reads the live bf16 mirror); later
        calls refresh the same copy in place, so its addresses, and any graph captured on it,
        stay valid.  The live model and the optimizer are only read."""
        if self.ema_decay is None:
            raise RuntimeError("ema_model: this TrainStep keeps no EMA (ema_decay=0)")
        if self._ema_model is None:
            m = copy.deepcopy(self.model)
            self._ema_pairs = list(zip(m.parameters(), self.model.parameters()))
            bufs = dict(m.named_buffers())
            self._ema_stats = [bufs[n] for n, _ in self.model.named_buffers()
                               if "running_mean" in n or "running_var" in n]
            self._ema_model = m
        with torch.no_grad():
            for q, p in self._ema_pairs:
                q.copy_(self.opt.ema_shadow(p))
            for b, s in zip(self._ema_stats, self.stat_shadow):
                b.copy_(s)
        return self._ema_model

    def validate(self, val_batches, calib_batches=None, calib_steps=None, calib_batch=None):
        """The reference's validate() (train.py:273-309): the EMA model, calibrated on
        `calib_batches` (at most `calib_steps` of them) when given, evaluated on `val_batches`.
        Returns {'loss', 'top1_error', 'top5_error'} (means over the samples of every rank)."""
        model = self.ema_model()
        if self._eval_step is None:
            self._eval_step = EvalStep(model, self.batch, image_size=self.x.shape[-1],
                                       calib_batch=calib_batch, use_graph=self.use_graph,
                                       input_dtype=self.x.dtype,
                                       input_norm=dataflow.input_norm_of(self.model),
                                       fused_multi_branch=self.fused_multi_branch)
        es = self._eval_step
        if calib_batches is not None:
            es.calibrate(calib_batches, calib_steps)
        return es.evaluate(val_batches)


def _attach_input_norm(model, input_dtype, input_norm):
    if input_dtype == torch.uint8 and input_norm is None:
        raise ValueError("uint8 input needs input_norm=(mean, std): the Normalize() of the "
                         "input pipeline, applied by the stem kernels")
    if input_norm is not None:
        dataflow.set_input_norm(model, *input_norm)


def ema_names(model):
    """(parameter names, running-statistics names) of `model`: together, the variables and the
    registration order of the reference's setup_ema (common.py:58-63); the second list is also
    the order of `TrainStep.stat_bufs`."""
    return ([n for n, _ in model.named_parameters()],
            [n for n, _ in model.named_buffers() if "running_mean" in n or "running_var" in n])


def ema_state_dict(shadow, num_updates, momentum):
    """The layout of the reference's ExponentialMovingAverage.state_dict() (utils/optim.py:87-95)
    for `shadow` ({name: fp32 tensor}, in registration order), every variable updated
    `num_updates` times with the momentum rule of `flat_arena.ema_momentum`."""
    last = ema_momentum(momentum, num_updates) if num_updates > 0 else None
    return {"info": OrderedDict((n, {"num_updates": num_updates, "last_momemtum": last,
                                     "zero_init": False}) for n in shadow),
            "shadow": OrderedDict(shadow),
            "param": {"momentum": momentum, "zero_debias": False}}


def metrics_from_sums(loss_sum, correct1, correct5, count):
    """The reference's validation results (forward_loss meters averaged over the samples,
    common.py:67-80) from the sums over every sample of every rank."""
    n = float(count)
    if n <= 0:
        raise ValueError("no samples were evaluated")
    return {"loss": float(loss_sum) / n, "top1_error": 1.0 - float(correct1) / n,
            "top5_error": 1.0 - float(correct5) / n}


class _Phase:
    """Static input buffers, staging copies and the captured graph of one EvalStep phase for its
    full batch shape."""

    def __init__(self, batch, image_size, dtype, dev):
        self.x = torch.zeros(batch, 3, image_size, image_size, device=dev,
                             dtype=dtype).contiguous(memory_format=torch.channels_last)
        self.t = torch.zeros(batch, dtype=torch.long, device=dev)
        self.x_stage = torch.zeros_like(self.x)
        self.t_stage = torch.zeros_like(self.t)
        self.graph = None
        self.warm = 0


class EvalStep:
    """Evaluation counterpart of TrainStep on the sm_90a path: bn_calibration and the validation
    pass of the reference (train.py:273-309) over a model that stays where it is (typically
    `TrainStep.ema_model()`).

    Each phase (calibration, evaluation) captures one CUDA graph for its full batch shape and
    replays it; a batch of another shape (a partial last batch) runs the same kernels eagerly.
    Everything weight-dependent (bf16 operands, folded BatchNorm coefficients, the classifier's
    bf16 bias) is recomputed inside the graph, so in-place weight updates between replays are
    seen.  A model whose parameters carry an optimizer's bf16 mirror needs that optimizer
    (`optimizer=`): its `sync_mirror()` runs before every replay.

    Evaluation sums the per-sample loss (fp64) and the correct@1 / correct@5 / sample counts
    (int64) on the device in batch order; there is no host sync per batch, and one all-reduce
    SUM at the end when the world is larger than one."""

    def __init__(self, model, per_gpu_batch, image_size=224, calib_batch=None, use_graph=True,
                 input_dtype=torch.bfloat16, optimizer=None, input_norm=None,
                 fused_multi_branch=False, small_batch=False):
        """`fused_multi_branch=True` runs the multi-branch blocks (several depthwise kernel sizes:
        AtomNAS) of the evaluation forwards as one packing launch and one block kernel each
        (engine.EVAL_MULTI_BRANCH) where engine.eval_mb_supported covers them.  Off by default: the
        hidden channels are regrouped by kernel size, so the project sums in another order and
        the logits differ from the default in the last bits (the same bits on every run).  A plain
        `model(x)` outside the step is not affected.

        `small_batch=True` (engine.EVAL_SMALL_BATCH) is for evaluation at a few images per batch
        (the searched networks at batch 1): multi-branch blocks split their hidden channels over a
        thread-block cluster, and the block kinds engine.SMALL_BATCH_FASTER lists run as one
        launch at batch sizes up to their measured bound.  Off by default, for the same reason;
        calibration and a plain `model(x)` are not affected."""
        _attach_input_norm(model, input_dtype, input_norm)
        dev = next(model.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("EvalStep needs the model on a CUDA device (no CPU path)")
        self.model = model
        self.dev = dev
        self.world = udist.get_world_size_fallback()
        self.optimizer = optimizer
        self.use_graph = use_graph
        self.fused_multi_branch = bool(fused_multi_branch)
        self.small_batch = bool(small_batch)
        self.phases = {"eval": _Phase(per_gpu_batch, image_size, input_dtype, dev),
                       "calib": _Phase(calib_batch or per_gpu_batch, image_size, input_dtype, dev)}
        self.loss_sum = torch.zeros((), device=dev, dtype=torch.float64)
        self.counts = torch.zeros(3, device=dev, dtype=torch.int64)   # correct@1, correct@5, samples
        self.logits = None           # logits of the last evaluated batch (fp32, device)
        self.copy_stream = torch.cuda.Stream(device=dev)
        self.copied = torch.cuda.Event()
        self.consumed = torch.cuda.Event()
        self.consumed.record()

    # ---- input path (as TrainStep.load) --------------------------------------------------------
    def load(self, x, target, phase="eval"):
        """Stage the next full batch of `phase` into its static buffers (async on the copy
        stream)."""
        ph = self.phases[phase]
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self.consumed)
            ph.x_stage.copy_(x, non_blocking=True)
            ph.t_stage.copy_(target, non_blocking=True)
            self.copied.record(self.copy_stream)

    def _publish(self, ph):
        cur = torch.cuda.current_stream()
        cur.wait_event(self.copied)
        ph.x.copy_(ph.x_stage)
        ph.t.copy_(ph.t_stage)
        self.consumed.record(cur)

    # ---- phase bodies ----------------------------------------------------------------------------
    def _calib_body(self, x, t):
        self.model(x)

    def _eval_body(self, x, t):
        engine.EVAL_TAIL_FUSED = True
        engine.EVAL_MULTI_BRANCH = self.fused_multi_branch
        engine.EVAL_SMALL_BATCH = self.small_batch
        try:
            logits = self.model(x)
        finally:
            engine.EVAL_TAIL_FUSED = False
            engine.EVAL_MULTI_BRANCH = False
            engine.EVAL_SMALL_BATCH = False
        loss, c1, c5 = tail_ops.softmax_ce(logits, t.to(self.dev), 0.0)
        self.loss_sum.add_(loss.double().sum())
        self.counts[0].add_(c1.sum().long())
        self.counts[1].add_(c5.sum().long())
        self.counts[2].add_(loss.shape[0])
        self.logits = logits

    def _run(self, phase, body, x, t):
        """One batch: a graph replay when it has the phase's full shape, else eagerly."""
        ph = self.phases[phase]
        if tuple(x.shape) != tuple(ph.x.shape):
            x = x.to(self.dev, non_blocking=True)
            if ph.x.dtype == torch.uint8:       # the stem normalises it
                x = x.contiguous(memory_format=torch.channels_last)
            else:
                x = engine.to_nhwc_bf16(x)
            body(x, t)
            return
        self.load(x, t, phase)
        self._publish(ph)
        if self.optimizer is not None:
            self.optimizer.sync_mirror()
        if self.use_graph and ph.graph is None and ph.warm >= 1:
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                body(ph.x, ph.t)
            ph.graph = g
            ph.logits = self.logits          # the eval graph's static output
        if ph.graph is not None:
            ph.graph.replay()
            if phase == "eval":
                self.logits = ph.logits
        else:
            body(ph.x, ph.t)
            ph.warm += 1

    # ---- the two phases --------------------------------------------------------------------------
    @torch.no_grad()
    def calibrate(self, batches, steps=None):
        """bn_calibration (reference utils/common.py:175-187, train.py:279-296): reset the
        running statistics of every nn.BatchNorm2d (ZeroInitBN included), give them momentum None
        (a cumulative average), put only them in train mode (a non-local InstanceNorm stays in
        eval mode), run `steps` forwards (all batches when None), all-reduce the statistics when
        the world is larger than one, and return the model to eval mode."""
        model = self.model
        model.eval()
        for m in model.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.reset_running_stats()
                m.momentum = None
                m.train()
        try:
            for i, (x, t) in enumerate(batches):
                if steps is not None and i >= steps:
                    break
                self._run("calib", self._calib_body, x, t)
        finally:
            model.eval()
        if self.world > 1:
            udist.allreduce_bn(model)

    @torch.no_grad()
    def evaluate(self, batches):
        """Eval pass (reference forward_loss with the plain cross entropy, common.py:67-80):
        returns {'loss', 'top1_error', 'top5_error'} over every sample of every rank.  The
        per-rank sums stay in `loss_sum` / `counts`."""
        self.model.eval()
        self.loss_sum.zero_()
        self.counts.zero_()
        for x, t in batches:
            self._run("eval", self._eval_body, x, t)
        if self.world > 1:
            dist.all_reduce(self.loss_sum)
            dist.all_reduce(self.counts)
        c = self.counts.tolist()
        return metrics_from_sums(float(self.loss_sum), c[0], c[1], c[2])
