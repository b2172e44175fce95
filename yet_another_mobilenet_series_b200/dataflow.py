"""Device-side input path with the surface of the reference's `DataPrefetcher`
(utils/dataflow.py:13-58): wrap any iterable of (input, target) host batches; the next batch is
copied to the GPU on a side stream while the current step computes, and `__next__` hands out
device tensors after making the compute stream wait for that copy.

Differences from the reference, all on the device side:
  * the batch lands directly in the layout and dtype the sm_90a kernels consume — bf16,
    channels_last — in ONE copy kernel (the reference uploads fp32 NCHW and calls `.float()`;
    its cuDNN path then converts per layer);
  * host batches should be pinned (`pin_memory=True` in the DataLoader) for the copy to overlap;
  * two device buffers are recycled instead of allocating a new tensor per batch, and an event
    (not a whole-stream wait) guards their reuse.
`TrainStep.load` is the same mechanism for a single static buffer (CUDA-graph replay).

uint8 input (the batches of NVIDIA apex's ImageNet example, the origin of the reference's
prefetcher): `fast_collate` packs decoded images as uint8 NCHW batches with channels_last storage,
`DataPrefetcher(loader, dtype=torch.uint8)` uploads them byte for byte (a quarter of the fp32
bytes), and a model given `set_input_norm(model, mean, std)` normalises them inside its stem
convolution kernels, to the bits `ToTensor()` + `Normalize(mean, std)` give on the host.
"""
import math

import numpy as np
import torch


def set_input_norm(model, mean, std):
    """Attach the `Normalize(mean, std)` of the input pipeline to `model` (the module whose forward
    runs the network, not a DDP wrapper): a uint8 image batch passed to it is then normalised by
    its stem kernels.  A plain attribute, not a buffer: state_dict() keys stay those of the
    reference, and copy.deepcopy (TrainStep.ema_model) carries it."""
    mean = tuple(float(v) for v in mean)
    std = tuple(float(v) for v in std)
    if len(mean) != 3 or len(std) != 3:
        raise ValueError("set_input_norm: mean and std need 3 values (RGB), got %r, %r" % (mean, std))
    if not all(math.isfinite(v) for v in mean + std) or any(v == 0.0 for v in std):
        raise ValueError("set_input_norm: mean and std must be finite and std non-zero: %r, %r"
                         % (mean, std))
    model.input_norm = (mean, std)
    return model


def input_norm_of(model):
    """The (mean, std) set_input_norm attached to `model`, or None."""
    return getattr(model, "input_norm", None)


def fast_collate(batch):
    """collate_fn for a DataLoader whose transforms end before `ToTensor()`: a list of
    (PIL RGB image or uint8 HWC array, target) -> (uint8 [N, 3, H, W] with channels_last storage,
    int64 [N]).  Each image is copied once, into one buffer, pinned when CUDA is available and
    the call runs in the main process (in DataLoader workers, use `pin_memory=True`: pinning
    there would initialise CUDA in a forked process)."""
    imgs = [np.asarray(img, dtype=np.uint8) for img, _ in batch]
    if not imgs:
        raise ValueError("fast_collate: empty batch")
    H, W = imgs[0].shape[:2]
    for a in imgs:
        if a.shape != (H, W, 3):
            raise ValueError("fast_collate: images must be RGB of one size, %r vs %r"
                             % (a.shape, (H, W, 3)))
    pin = torch.cuda.is_available() and torch.utils.data.get_worker_info() is None
    out = torch.empty((len(imgs), H, W, 3), dtype=torch.uint8, pin_memory=pin)
    dst = out.numpy()
    for i, a in enumerate(imgs):
        dst[i] = a
    target = torch.tensor([int(t) for _, t in batch], dtype=torch.int64)
    return out.permute(0, 3, 1, 2), target


class DataPrefetcher:
    def __init__(self, loader, device=None, dtype=torch.bfloat16):
        if not torch.cuda.is_available():
            raise RuntimeError("DataPrefetcher needs a CUDA device (it IS the device-side input path)")
        self.loader_len = len(loader) if hasattr(loader, "__len__") else None
        self.loader = iter(loader)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else device
        self.dtype = dtype
        self.stream = torch.cuda.Stream(device=self.device)
        self.bufs = [None, None]        # recycled (input, target) device buffers
        self.free = [torch.cuda.Event(), torch.cuda.Event()]
        self.slot = 0
        self.handed = None              # slot the caller is currently computing on
        self.stop = False
        self.preload()

    def preload(self):
        try:
            x, t = next(self.loader)
        except StopIteration:
            self.stop = True
            self.next_input = self.next_target = None
            return
        s = self.slot
        buf = self.bufs[s]
        if buf is None or buf[0].shape != x.shape or buf[1].shape != t.shape:
            buf = (torch.empty(x.shape, device=self.device, dtype=self.dtype).contiguous(
                       memory_format=torch.channels_last if x.dim() == 4 else torch.contiguous_format),
                   torch.empty(t.shape, device=self.device, dtype=t.dtype))
            self.bufs[s] = buf
        with torch.cuda.stream(self.stream):
            self.stream.wait_event(self.free[s])          # the consumer is done with this slot
            buf[0].copy_(x, non_blocking=True)            # H2D + fp32->bf16 + NCHW->NHWC in one pass
            buf[1].copy_(t, non_blocking=True)
        self.next_input, self.next_target = buf
        self.next_slot = s
        self.slot = 1 - s

    def __next__(self):
        if self.stop:
            raise StopIteration
        cur = torch.cuda.current_stream(self.device)
        cur.wait_stream(self.stream)
        # everything the caller enqueued on the batch handed out LAST time is in the stream by now:
        # from this point on that slot may be refilled (the preload below targets exactly it)
        if self.handed is not None:
            self.free[self.handed].record(cur)
        x, t, s = self.next_input, self.next_target, self.next_slot
        self.handed = s
        self.preload()
        return x, t

    def __iter__(self):
        return self

    def __len__(self):
        return self.loader_len
