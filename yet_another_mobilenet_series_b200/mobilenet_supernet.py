"""MobileNetV2-style network builder with the surface of the reference's
`models/mobilenet_supernet.py` (:59-176): same constructor keywords (so
`apps/mobilenet/models/*.yml` load unchanged through `model: <this module>`,
reference common.py:129-130), same module tree / state_dict keys.  The inverted-residual blocks
come from `mobilenet_base.get_block` and run on the sm_90a kernels; activations flow between
blocks as channels_last bf16."""
import numbers

import torch
from torch import nn

from .mobilenet_base import ConvBNReLU, _make_divisible, get_active_fn, get_block
from . import engine
from .dataflow import input_norm_of

__all__ = ["MobileNetV2"]


def _hidden_dims(inp, expand_ratio, kernel_sizes):
    """Expand ratio(s) -> per-branch hidden widths (reference :31-42)."""
    if isinstance(expand_ratio, list):
        assert len(expand_ratio) == len(kernel_sizes)
        ratios, expand = expand_ratio, True
    elif isinstance(expand_ratio, numbers.Number):
        ratios, expand = [expand_ratio] * len(kernel_sizes), expand_ratio != 1
    else:
        raise ValueError("Unknown expand_ratio type: {}".format(expand_ratio))
    return [int(round(inp * r)) for r in ratios], expand


def get_block_wrapper(block_str):
    """Block class taking `expand_ratio` instead of explicit hidden widths (reference :13-56)."""
    base = get_block(block_str)

    class InvertedResidual(base):

        def __init__(self, inp, oup, stride, expand_ratio, kernel_sizes, active_fn=None,
                     batch_norm_kwargs=None, **kwargs):
            hidden, expand = _hidden_dims(inp, expand_ratio, kernel_sizes)
            super().__init__(inp, oup, stride, hidden, kernel_sizes, expand, active_fn=active_fn,
                             batch_norm_kwargs=batch_norm_kwargs, **kwargs)
            self.expand_ratio = expand_ratio

    return InvertedResidual


def _full_extent(pool, x):
    k = pool.kernel_size if isinstance(pool.kernel_size, tuple) else (pool.kernel_size,) * 2
    st = pool.stride if isinstance(pool.stride, tuple) else (pool.stride,) * 2
    pad = pool.padding if isinstance(pool.padding, tuple) else (pool.padding,) * 2
    return tuple(x.shape[2:]) == tuple(k) and tuple(st) == tuple(k) and tuple(pad) == (0, 0)


# ---- instrumentation (model_profiling) -----------------------------------------------------------
# When STEPS is a list, run_features on CUDA records a CUDA event on the current stream before its
# first step and after each one, and appends (module, event): (None, e) first, then the stem (its
# step includes the input's conversion to bf16 channels_last), each block, the head, the pool and
# model.classifier (its step includes the cast of the logits to fp32).  The time between two
# consecutive events is the device time of the step the second one ends.  A head run together with
# the pool (engine.EVAL_TAIL_FUSED, engine.TRAIN_TAIL_FUSED) is one step, recorded for the head; a
# stem run together with the first block (engine.TRAIN_STEM_FUSED) is one step, recorded for the
# stem.
STEPS = None


def _step_done(stream, module):
    """Ends `module`'s step on `stream`, the current stream looked up once per forward (the lookup
    costs the host more than the record); None when STEPS is off."""
    if stream is not None:
        e = torch.cuda.Event(enable_timing=True)
        e.record(stream)
        STEPS.append((module, e))


def run_features(model, x):
    """Shared forward of both builders: bf16 channels_last through stem, blocks, head, pool.  A
    uint8 image on a model with an input normalisation (dataflow.set_input_norm) goes to the stem
    as it is; the stem normalises it."""
    if x.is_cuda:
        from . import tail_ops
        stream = torch.cuda.current_stream() if STEPS is not None else None
        _step_done(stream, None)
        norm = input_norm_of(model) if x.dtype == torch.uint8 else None
        if norm is None:
            x = engine.to_nhwc_bf16(x)
        else:
            x = x.contiguous(memory_format=torch.channels_last)
        layers = list(model.features)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            skip = False
            for i, layer in enumerate(layers):
                if skip:
                    skip = False
                    continue
                nxt = layers[i + 1] if i + 1 < len(layers) else None
                if (i == 0 and engine.TRAIN_STEM_FUSED and nxt is not None
                        and tail_ops.stem_block_fused_covered(layer, nxt, x)):
                    # training: stem ConvBNReLU + its only consumer, the first block, as one
                    # autograd function (the stem's BatchNorm + activation inside the depthwise)
                    x, skip = tail_ops.stem_block_train(layer, nxt, x, norm), True
                    _step_done(stream, layer)
                    continue
                if i == 0 and norm is not None:
                    x = tail_ops.stem_u8(layer, x, norm)
                    _step_done(stream, layer)
                    continue
                if ((engine.EVAL_TAIL_FUSED or engine.TRAIN_TAIL_FUSED)
                        and isinstance(layer, ConvBNReLU)
                        and isinstance(nxt, nn.AvgPool2d) and _full_extent(nxt, x)):
                    # head 1x1 ConvBNReLU + global average pool: in eval one launch, in training
                    # the head GEMM + one pooling kernel (when covered)
                    y = tail_ops.head_pool_eval(layer, x) if engine.EVAL_TAIL_FUSED else None
                    if y is None and engine.TRAIN_TAIL_FUSED:
                        y = tail_ops.head_pool_train(layer, x)
                    if y is not None:
                        x, skip = y, True
                        _step_done(stream, layer)
                        continue
                if (isinstance(layer, nn.AvgPool2d) and _full_extent(layer, x)):
                    # global average pool: same numbers as nn.AvgPool2d(H), but torch's NHWC
                    # avg_pool2d backward kernel took 0.24 ms for this 16 M-element tensor
                    x = x.mean((2, 3), keepdim=True)
                else:
                    x = layer(x)
                _step_done(stream, layer)
            x = x.flatten(1)
            x = run_classifier(model.classifier, x)
        x = x.float()
        _step_done(stream, model.classifier)
        return x
    # CPU: stem/head/classifier are plain torch, but the blocks have no CPU path and will raise
    x = model.features(x)
    return model.classifier(x.squeeze(3).squeeze(2))


def run_classifier(classifier, x):
    """Dropout -> Linear (reference :163-167); the Linear runs on the wgmma GEMM when its
    widths allow (tail_ops.linear_apply), else as the torch module."""
    from . import tail_ops
    for layer in classifier:
        if isinstance(layer, nn.Linear) and tail_ops.linear_supported(layer, x):
            x = tail_ops.linear_apply(layer, x)
        else:
            x = layer(x)
    return x


class MobileNetV2(nn.Module):
    """MobileNetV2-like network (reference :59-173); rows are
    `[t, c, n, s, ks]` or `[t, c, n, s, ks, nl_c, nl_s, se_ratio]`."""

    def __init__(self, num_classes=1000, input_size=224, input_channel=32, last_channel=1280,
                 width_mult=1.0, inverted_residual_setting=None, dropout_ratio=0.2,
                 batch_norm_momentum=0.1, batch_norm_epsilon=1e-5, active_fn="nn.ReLU6",
                 block="InvertedResidualChannels", round_nearest=8):
        super().__init__()
        bn_kw = {"momentum": batch_norm_momentum, "eps": batch_norm_epsilon}
        self.input_channel = input_channel
        self.last_channel = last_channel
        self.width_mult = width_mult
        self.round_nearest = round_nearest
        self.inverted_residual_setting = inverted_residual_setting
        self.active_fn = active_fn
        self.block = block
        rows = inverted_residual_setting
        if len(rows) == 0 or len(rows[0]) not in [5, 8]:
            raise ValueError("inverted_residual_setting should be non-empty "
                             "or a 5/8-element list, got {}".format(rows))
        if input_size % 32 != 0:
            raise ValueError("Input size must divide 32")
        act = get_active_fn(active_fn)
        block_cls = get_block_wrapper(block)
        width = _make_divisible(input_channel * width_mult, round_nearest)
        last = _make_divisible(last_channel * max(1.0, width_mult), round_nearest)
        layers = [ConvBNReLU(3, width, stride=2, batch_norm_kwargs=bn_kw, active_fn=act)]
        for t, c, n, s, ks, *extra in rows:
            out = _make_divisible(c * width_mult, round_nearest)
            kw = dict(zip(["nl_c", "nl_s", "se_ratio"], extra)) if len(extra) == 3 else {}
            for i in range(n):
                layers.append(block_cls(width, out, s if i == 0 else 1, t, ks, active_fn=act,
                                        batch_norm_kwargs=bn_kw, **kw))
                width = out
        layers.append(ConvBNReLU(width, last, kernel_size=1, batch_norm_kwargs=bn_kw,
                                 active_fn=act))
        layers.append(nn.AvgPool2d(input_size // 32))
        self.features = nn.Sequential(*layers)
        self.classifier = nn.Sequential(nn.Dropout(dropout_ratio), nn.Linear(last, num_classes))

    def forward(self, x):
        return run_features(self, x)


Model = MobileNetV2
