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
"""
import torch


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
