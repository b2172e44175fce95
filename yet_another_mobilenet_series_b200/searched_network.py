"""Searched-network builder with the surface of the reference's `models/searched_network.py`
(:13-139): rows are `[c, n, s, ks, hiddens, expand]` with explicit hidden widths, optional global
`se_ratio` (fused block only).  Same module tree / state_dict keys; blocks run on sm_90a."""
import warnings

from torch import nn

from .mobilenet_base import ConvBNReLU, InvertedResidualChannelsFused, get_active_fn, get_block
from .mobilenet_supernet import run_features

__all__ = ["MobileNetSearched"]


class MobileNetSearched(nn.Module):

    def __init__(self, num_classes=1000, input_size=224, input_channel=32, last_channel=1280,
                 width_mult=1.0, inverted_residual_setting=None, dropout_ratio=0.2, se_ratio=None,
                 batch_norm_momentum=0.1, batch_norm_epsilon=1e-5, active_fn="nn.ReLU6",
                 block="InvertedResidualChannels", round_nearest=8):
        super().__init__()
        bn_kw = {"momentum": batch_norm_momentum, "eps": batch_norm_epsilon}
        if width_mult != 1.0:
            raise ValueError("Searched model should have width 1")
        self.input_channel = input_channel
        self.last_channel = last_channel
        self.width_mult = width_mult
        self.round_nearest = round_nearest
        self.inverted_residual_setting = inverted_residual_setting
        self.active_fn = active_fn
        self.block = block
        rows = inverted_residual_setting
        if len(rows) == 0 or len(rows[0]) != 6:
            raise ValueError("inverted_residual_setting should be non-empty "
                             "or a 6-element list, got {}".format(rows))
        if input_size % 32 != 0:
            raise ValueError("Input size must divide 32")
        for name, channel in (("Input", input_channel), ("Last", last_channel)):
            if (channel * width_mult) % round_nearest:
                warnings.warn("{} channel could not divide {}".format(name, round_nearest))
        act = get_active_fn(active_fn)
        block_cls = get_block(block)
        extra = {}
        if se_ratio is not None:
            if not issubclass(block_cls, InvertedResidualChannelsFused):
                raise NotImplementedError(
                    "SE module not supported for block: {}".format(block_cls))
            extra["se_ratio"] = se_ratio
        width = input_channel
        layers = [ConvBNReLU(3, width, stride=2, batch_norm_kwargs=bn_kw, active_fn=act)]
        for c, n, s, ks, hiddens, expand in rows:
            for i in range(n):
                layers.append(block_cls(width, c, s if i == 0 else 1, hiddens, ks, expand,
                                        active_fn=act, batch_norm_kwargs=bn_kw, **extra))
                width = c
        layers.append(ConvBNReLU(width, last_channel, kernel_size=1, batch_norm_kwargs=bn_kw,
                                 active_fn=act))
        layers.append(nn.AvgPool2d(input_size // 32))
        self.features = nn.Sequential(*layers)
        self.classifier = nn.Sequential(nn.Dropout(dropout_ratio),
                                        nn.Linear(last_channel, num_classes))

    def forward(self, x):
        return run_features(self, x)


Model = MobileNetSearched
