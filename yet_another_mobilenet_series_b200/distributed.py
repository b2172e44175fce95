"""Data-parallel plumbing with the surface of the reference's `utils/distributed.py`, one process
per GPU over NCCL (NVLink / NVSwitch inside one node).

The data path of the reference has exactly one exchange step per iteration: the SUM all-reduce of
all gradients followed by a division by the world size (utils/distributed.py:131-139, called from
train.py:72-73).  Here the gradients already live in ONE flat fp32 arena (fused_rmsprop.RMSprop, fused_sgd.SGD),
so `allreduce_grads` is a single in-place NCCL all-reduce with no flatten / unflatten copies, and
the division is folded into the optimizer kernel (`grad_scale`).  BatchNorm statistics stay local
during training, like the reference (`allreduce_bn: False` in every training yml).

Mirrored API: init_dist :25-32, is_master :51-53, get_rank_fallback / get_world_size_fallback
:56-69, master_only :71-80, allreduce_grads :155-161, allreduce_bn :164-169,
AllReduceDistributedDataParallel :172-199.
"""
import functools
import os

import torch
import torch.distributed as dist
from torch import nn


def _get_env(name):
    if name not in os.environ:
        raise RuntimeError("${} should be set".format(name))
    return os.environ[name]


def init_dist(backend="nccl", **kwargs):
    """One process per GPU: bind LOCAL_RANK's device, join the process group (env:// rendezvous)."""
    if dist.is_initialized():
        raise RuntimeError("Should not init distributed twice")
    rank = int(_get_env("RANK"))
    local_rank = int(_get_env("LOCAL_RANK"))
    if backend == "nccl":
        assert rank % torch.cuda.device_count() == local_rank
        torch.cuda.set_device(local_rank)
        kwargs.setdefault("device_id", torch.device("cuda", local_rank))
    dist.init_process_group(backend=backend, **kwargs)


def get_rank_fallback():
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def get_world_size_fallback():
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def is_master():
    return get_rank_fallback() == 0


def master_only(func):
    @functools.wraps(func)
    def wrapper(*args, **kwargs):
        return func(*args, **kwargs) if is_master() else None
    return wrapper


def _flat_allreduce(tensors, average=True):
    """Generic coalesced all-reduce (one flat buffer per dtype) for tensors that are not already
    views of one arena: BN running statistics, foreign optimizers."""
    world = get_world_size_fallback()
    if world < 2 or not tensors:
        return
    by_type = {}
    for t in tensors:
        by_type.setdefault(t.dtype, []).append(t)
    for group in by_type.values():
        flat = torch.cat([t.reshape(-1) for t in group])
        dist.all_reduce(flat)
        if average:
            flat.div_(world)
        off = 0
        for t in group:
            n = t.numel()
            t.copy_(flat[off:off + n].view_as(t))
            off += n


def allreduce_grads(model, optimizer=None, defer_mean=False):
    """Mean of the gradients over ranks (reference :155-161).

    With the flat-arena optimizer the all-reduce runs IN PLACE on the arena; `defer_mean=True`
    leaves the SUM in the arena and sets `optimizer.grad_scale = 1/world` so the division happens
    inside the fused step kernel."""
    world = get_world_size_fallback()
    arenas = optimizer.arenas() if optimizer is not None and hasattr(optimizer, "arenas") else None
    if arenas is not None:
        if world > 1:
            dist.all_reduce(arenas["g"])
        if defer_mean:
            optimizer.grad_scale = 1.0 / world
        elif world > 1:
            arenas["g"].div_(world)
        return
    grads = [p.grad.data for p in model.parameters() if p.requires_grad and p.grad is not None]
    _flat_allreduce(grads)


def allreduce_bn(model):
    """Average BatchNorm running statistics over ranks (reference :164-169; used after
    calibration, train.py:295-296)."""
    bufs = [b for n, b in model.named_buffers() if "running_var" in n or "running_mean" in n]
    _flat_allreduce(bufs)


class AllReduceDistributedDataParallel(nn.Module):
    """Wrapper of the reference (:172-199): broadcast rank 0's parameters and buffers at
    construction, no gradient hooks (the trainer calls `allreduce_grads` explicitly)."""

    def __init__(self, module, dim=0, broadcast_buffers=True, bucket_cap_mb=25):
        super().__init__()
        self.module = module
        self.dim = dim
        self.broadcast_buffers = broadcast_buffers
        self.broadcast_bucket_size_mb = bucket_cap_mb
        self._sync_params()

    def _sync_params(self):
        if get_world_size_fallback() < 2:
            return
        states = list(self.module.state_dict().values())
        if self.broadcast_buffers:
            states += [b.data for b in self.module.buffers()]
        for t in states:
            dist.broadcast(t, 0)
        # the broadcast wrote the fp32 masters through detached views: if a fused optimizer already
        # keeps a bf16 mirror of them (the tensor-core operand), re-cast it now (ADVICE r1)
        with torch.no_grad():
            for p in self.module.parameters():
                mirror = getattr(p, "_yamb_bf16", None)
                if mirror is not None:
                    mirror.copy_(p)
                    p._yamb_bf16_version = p._version

    def forward(self, *inputs, **kwargs):
        return self.module(*inputs, **kwargs)
