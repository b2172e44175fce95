"""Block library with the module surface of the reference's `models/mobilenet_base.py`, backed by
the sm_90a kernels.

Drop-in contract (SURVEY.md §8b): same class names, constructor signatures, attributes, child
module names and therefore the same `state_dict()` keys/shapes, the same helper methods
(`get_depthwise_bn`, `get_named_depthwise_bn`), `__repr__` formats and registries
(`get_block`, `get_active_fn`, `get_nl_norm_fn`) as

  InvertedResidualChannels        /root/reference/models/mobilenet_base.py:352-458
  InvertedResidualChannelsFused   /root/reference/models/mobilenet_base.py:206-349
  ConvBNReLU :181-203, SqueezeAndExcitation :91-118, Nonlocal :131-178, ZeroInitBN :121-128,
  Swish :70-78, HSwish :81-88, Narrow/Identity :50-67, init_weights_* :492-537

so the reference's yml model descriptions, checkpoints, `bn_calibration`, `cal_l2_loss`,
`setup_ema` and the profiler (which all reach into the children) work unchanged.  The children
stay real `nn.Conv2d` / `nn.BatchNorm2d` parameter holders; only `forward` of the two block
classes is replaced: on CUDA it runs the fused kernel sequence of `engine.py`
(there is no CPU fallback for it).
"""
import collections
import functools
import logging
import math

import torch
from torch import nn
from torch.nn import functional as F

from . import engine


def add_prefix(name, prefix=None, split="."):
    """`prefix.name` when a prefix is given (reference utils/common.py:159-164)."""
    return name if prefix is None else "{}{}{}".format(prefix, split, name)


def _make_divisible(v, divisor, min_value=None):
    """Round `v` to a multiple of `divisor`, never dropping more than 10 %
    (reference :15-29; the rule of the TF-slim MobileNet)."""
    floor = divisor if min_value is None else min_value
    rounded = int(v + divisor / 2) // divisor * divisor
    rounded = max(floor, rounded)
    return rounded + divisor if rounded < 0.9 * v else rounded


class Identity(nn.Module):
    """No-op placeholder (reference :50-54)."""

    def forward(self, x):
        return x


class Narrow(nn.Module):
    """`x.narrow(dimension, start, length)` as a module (reference :57-67)."""

    def __init__(self, dimension, start, length):
        super().__init__()
        self.dimension, self.start, self.length = dimension, start, length

    def forward(self, x):
        return torch.narrow(x, self.dimension, self.start, self.length)


class Swish(nn.Module):
    """x * sigmoid(x) (reference :70-78)."""

    def forward(self, x):
        return torch.sigmoid(x) * x


class HSwish(nn.Module):
    """x * relu6(x + 3) / 6.  The reference's class (:81-88) is a plain `object` that
    `nn.Sequential` rejects (SURVEY.md §0); this is the same math as a working module —
    an extension, not a parity item."""

    def forward(self, x):
        return x * F.relu6(x + 3.0) / 6.0


class SqueezeAndExcitation(nn.Module):
    """Channel gating: x * sigmoid(W_e act(W_r mean_HW(x) + b_r) + b_e) (reference :91-118)."""

    def __init__(self, n_feature, n_hidden, spatial_dims=[2, 3], active_fn=None):
        super().__init__()
        self.n_feature = n_feature
        self.n_hidden = n_hidden
        self.spatial_dims = spatial_dims
        self.se_reduce = nn.Conv2d(n_feature, n_hidden, 1, bias=True)
        self.se_expand = nn.Conv2d(n_hidden, n_feature, 1, bias=True)
        self.active_fn = active_fn()

    def forward(self, x):
        pooled = x.mean(self.spatial_dims, keepdim=True)
        gate = torch.sigmoid(self.se_expand(self.active_fn(self.se_reduce(pooled))))
        return gate * x

    def __repr__(self):
        return "{}({}, {}, spatial_dims={}, active_fn={})".format(
            self._get_name(), self.n_feature, self.n_hidden, self.spatial_dims, self.active_fn)


class ZeroInitBN(nn.BatchNorm2d):
    """BatchNorm2d whose affine parameters start at zero (reference :121-128)."""

    def reset_parameters(self):
        self.reset_running_stats()
        if self.affine:
            nn.init.zeros_(self.weight)
            nn.init.zeros_(self.bias)


class Nonlocal(nn.Module):
    """Lightweight non-local block (reference :131-178): parameter holder with the reference's
    module tree (`depthwise_conv`, `bn`).  Inside a fused block on CUDA its arithmetic runs in the
    block's kernel sequence (engine.BlockPlan._nl_forward / _nl_backward: yamb_nl_gram,
    yamb_nl_rowmat, the depthwise and BatchNorm kernels); this `forward` is the stand-alone
    stock-torch statement of the same function (CPU, oracle, `as_reference`).

    `nl_norm`: the reference reads it from its global FLAGS inside the constructor (:151, "TODO:
    as param").  Here it is a keyword; when the reference's `utils.config` is already loaded in
    the process (its train.py imported this package through `model:`) and defines `nl_norm`, that
    value is honoured exactly as the reference would."""

    def __init__(self, n_feature, nl_c, nl_s, batch_norm_kwargs=None, nl_norm=None):
        super().__init__()
        self.n_feature, self.nl_c, self.nl_s = n_feature, nl_c, nl_s
        if nl_norm is None:
            import sys
            cfg = sys.modules.get("utils.config")     # never trigger its argv-parsing import
            flags = getattr(cfg, "FLAGS", None) if cfg is not None else None
            if flags is not None and hasattr(flags, "nl_norm"):
                nl_norm = flags.nl_norm
        self.depthwise_conv = nn.Conv2d(n_feature, n_feature, 3, 1, 1, groups=n_feature,
                                        bias=False)
        kw = {} if batch_norm_kwargs is None else batch_norm_kwargs
        norm = ZeroInitBN if nl_norm is None else get_nl_norm_fn(nl_norm)
        self.bn = norm(n_feature, **kw)

    def forward(self, l):
        N, C, H, W = l.shape
        s = self.nl_s
        c_red = int(self.nl_c * C)
        sub = l[:, :, ::s, ::s]
        theta, phi, g = l[:, :c_red], sub[:, :c_red], sub
        hw, hw_r = H * W, (H // s) * (W // s)
        # pick the cheaper association order, as the reference does (:164-170)
        if hw * hw_r * C * (1 + self.nl_c) < hw * C ** 2 * self.nl_c + hw_r * C ** 2 * self.nl_c:
            f = torch.einsum("niab,nicd->nabcd", theta, phi)
            f = torch.einsum("nabcd,nicd->niab", f, g)
        else:
            f = torch.einsum("nihw,njhw->nij", phi, g)
            f = torch.einsum("nij,nihw->njhw", f, theta)
        f = f / H * W  # sic: (f / H) * W, kept for parity (:171)
        return self.bn(self.depthwise_conv(f)) + l

    def __repr__(self):
        return "{}({}, nl_c={}, nl_s={}".format(self._get_name(), self.n_feature, self.nl_c,
                                                self.nl_s)


class ConvBNReLU(nn.Sequential):
    """conv(bias=False, pad=(k-1)//2) -> BatchNorm2d -> activation (reference :181-203)."""

    def __init__(self, in_planes, out_planes, kernel_size=3, stride=1, groups=1, active_fn=None,
                 batch_norm_kwargs=None):
        kw = {} if batch_norm_kwargs is None else batch_norm_kwargs
        super().__init__(
            nn.Conv2d(in_planes, out_planes, kernel_size, stride, (kernel_size - 1) // 2,
                      groups=groups, bias=False),
            nn.BatchNorm2d(out_planes, **kw),
            active_fn())

    def forward(self, x):
        # CUDA: a 1x1 convolution (the head 320 -> 1280) is the blocks' wgmma GEMM with the
        # BatchNorm statistics in its epilogue (tail_ops.pw_conv_bn_act); the 3x3 stride-2 stem
        # runs the direct kernels of tail_ops.stem_conv_bn_act; any other convolution stays a
        # library call with BatchNorm + activation on this repo's kernels.  CPU / odd widths: the
        # plain torch modules.
        conv, bn, act = self[0], self[1], self[2]
        from . import tail_ops
        if tail_ops.pw_conv_supported(self, x):
            return tail_ops.pw_conv_bn_act(self, x)
        if tail_ops.stem_supported(self, x):
            return tail_ops.stem_conv_bn_act(self, x)
        if (x.is_cuda and conv.groups == 1 and bn.num_features % 8 == 0 and bn.affine
                and type(act).__name__ in ("ReLU", "ReLU6", "Swish", "HSwish", "Identity")):
            return engine.bn_act_apply(bn, act, conv(x))
        return super().forward(x)


def _depthwise_stage(hidden, k, stride, active_fn, bn_kw):
    return ConvBNReLU(hidden, hidden, kernel_size=k, stride=stride, groups=hidden,
                      active_fn=active_fn, batch_norm_kwargs=bn_kw)


class _FusedBlockBase(nn.Module):
    """Shared behaviour of the two block packings: CUDA forward through the kernel engine."""

    def _check_ctor(self, stride, channels, kernel_sizes):
        assert stride in [1, 2]
        assert len(channels) == len(kernel_sizes)

    def forward(self, x):
        return engine.block_apply(self, x)

    def __deepcopy__(self, memo):
        # plans hold device buffers keyed to this instance; a copy (e.g. the EMA model,
        # reference common.py:164) must build its own
        import copy
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k in ("_yamb_plans", "_yamb_shadow", "_yamb_eval"):
                continue
            setattr(new, k, copy.deepcopy(v, memo))
        return new

    def get_depthwise_bn(self):
        """BatchNorm modules that follow the depthwise convolutions."""
        return list(self.get_named_depthwise_bn().values())


class InvertedResidualChannelsFused(_FusedBlockBase):
    """One expand conv for all branches, per-branch depthwise, optional SE / non-local
    (reference :206-349)."""

    def __init__(self, inp, oup, stride, channels, kernel_sizes, expand, active_fn=None,
                 batch_norm_kwargs=None, se_ratio=None, nl_c=0, nl_s=0):
        super().__init__()
        self._check_ctor(stride, channels, kernel_sizes)
        self.input_dim, self.output_dim = inp, oup
        self.expand, self.stride = expand, stride
        self.kernel_sizes, self.channels = kernel_sizes, channels
        self.use_res_connect = self.stride == 1 and inp == oup
        self.batch_norm_kwargs = batch_norm_kwargs
        self.active_fn = active_fn
        self.se_ratio, self.nl_c, self.nl_s = se_ratio, nl_c, nl_s
        (self.expand_conv, self.depth_ops, self.project_conv, self.se_op,
         self.nl_op) = self._build(channels, kernel_sizes, expand, se_ratio, nl_c, nl_s)

    def _build(self, hidden_dims, kernel_sizes, expand, se_ratio, nl_c, nl_s):
        bn_kw = self.batch_norm_kwargs if self.batch_norm_kwargs is not None else {}
        total = sum(hidden_dims)
        expand_conv = ConvBNReLU(self.input_dim, total, kernel_size=1, batch_norm_kwargs=bn_kw,
                                 active_fn=self.active_fn) if self.expand else Identity()
        depth_ops = nn.ModuleList()
        offset = 0
        for k, hidden in zip(kernel_sizes, hidden_dims):
            stage = []
            if expand:
                stage.append(Narrow(1, offset, hidden))
                offset += hidden
            else:
                if hidden != self.input_dim:
                    raise RuntimeError("uncomment this for search_first model")
                logging.warning("uncomment this for previous trained search_first model")
            stage.append(_depthwise_stage(hidden, k, self.stride, self.active_fn, bn_kw))
            depth_ops.append(nn.Sequential(*stage))
        project_conv = nn.Sequential(nn.Conv2d(total, self.output_dim, 1, 1, 0, bias=False),
                                     nn.BatchNorm2d(self.output_dim, **bn_kw))
        if expand and offset != total:
            raise ValueError("Part of expanded are not used")
        if se_ratio is not None and se_ratio > 0:
            se_op = SqueezeAndExcitation(total, int(round(self.input_dim * se_ratio)),
                                         active_fn=self.active_fn)
        else:
            se_op = Identity()
        nl_op = Nonlocal(self.output_dim, nl_c, nl_s, batch_norm_kwargs=bn_kw) if nl_c > 0 \
            else Identity()
        return expand_conv, depth_ops, project_conv, se_op, nl_op

    def get_named_depthwise_bn(self, prefix=None):
        """`{name: BatchNorm2d}` keyed `depth_ops.{i}.1.1` (pinned by the reference's
        tests/models/mobilenet_base_test.py:55-64)."""
        if not self.expand:
            raise RuntimeError("Not search_first")
        found = collections.OrderedDict()
        for i, op in enumerate(self.depth_ops):
            stage = list(op.children())[1]
            assert isinstance(stage, ConvBNReLU)
            bn = stage[1]
            assert isinstance(bn, nn.BatchNorm2d)
            found[add_prefix("depth_ops.{}.{}.1".format(i, 1), prefix)] = bn
        return found

    def __repr__(self):
        return ("{}({}, {}, channels={}, kernel_sizes={}, expand={}, stride={},"
                " se_ratio={}, nl_s={}, nl_c={})").format(
                    self._get_name(), self.input_dim, self.output_dim, self.channels,
                    self.kernel_sizes, self.expand, self.stride, self.se_ratio, self.nl_s,
                    self.nl_c)


class InvertedResidualChannels(_FusedBlockBase):
    """Per-branch expand -> depthwise -> project, summed, then `pw_bn` (reference :352-458)."""

    def __init__(self, inp, oup, stride, channels, kernel_sizes, expand, active_fn=None,
                 batch_norm_kwargs=None):
        super().__init__()
        self._check_ctor(stride, channels, kernel_sizes)
        self.input_dim, self.output_dim = inp, oup
        self.expand, self.stride = expand, stride
        self.kernel_sizes, self.channels = kernel_sizes, channels
        self.use_res_connect = self.stride == 1 and inp == oup
        self.batch_norm_kwargs = batch_norm_kwargs
        self.active_fn = active_fn
        self.ops, self.pw_bn = self._build(channels, kernel_sizes, expand)

    def _build(self, hidden_dims, kernel_sizes, expand):
        bn_kw = self.batch_norm_kwargs if self.batch_norm_kwargs is not None else {}
        ops = nn.ModuleList()
        consumed = 0
        for k, hidden in zip(kernel_sizes, hidden_dims):
            stage = []
            if expand:
                stage.append(ConvBNReLU(self.input_dim, hidden, kernel_size=1,
                                        batch_norm_kwargs=bn_kw, active_fn=self.active_fn))
            else:
                if hidden != self.input_dim:
                    raise RuntimeError("uncomment this for search_first model")
                logging.warning("uncomment this for previous trained search_first model")
                consumed += hidden
            stage.append(_depthwise_stage(hidden, k, self.stride, self.active_fn, bn_kw))
            stage.append(nn.Conv2d(hidden, self.output_dim, 1, 1, 0, bias=False))
            ops.append(nn.Sequential(*stage))
        pw_bn = nn.BatchNorm2d(self.output_dim, **bn_kw)
        if not expand and consumed != self.input_dim:
            raise ValueError("Part of input are not used")
        return ops, pw_bn

    def get_named_depthwise_bn(self, prefix=None):
        """`{name: BatchNorm2d}` keyed `ops.{i}.{1|0}.1` (pinned by the reference's
        tests/models/mobilenet_base_test.py:26-35)."""
        where = 1 if self.expand else 0
        found = collections.OrderedDict()
        for i, op in enumerate(self.ops):
            stage = list(op.children())[where]
            assert isinstance(stage, ConvBNReLU)
            bn = stage[1]
            assert isinstance(bn, nn.BatchNorm2d)
            found[add_prefix("ops.{}.{}.1".format(i, where), prefix)] = bn
        return found

    def __repr__(self):
        return ("{}({}, {}, channels={}, kernel_sizes={}, expand={},"
                " stride={})").format(self._get_name(), self.input_dim, self.output_dim,
                                      self.channels, self.kernel_sizes, self.expand, self.stride)


_ACTIVE_FNS = {
    "nn.ReLU6": functools.partial(nn.ReLU6, inplace=True),
    "nn.ReLU": functools.partial(nn.ReLU, inplace=True),
    "nn.Swish": Swish,
    "nn.HSwish": HSwish,
}
_NL_NORMS = {
    "nn.BatchNorm": ZeroInitBN,
    "nn.InstanceNorm": functools.partial(nn.InstanceNorm2d, affine=True,
                                         track_running_stats=True),
}
_BLOCKS = {
    "InvertedResidualChannels": InvertedResidualChannels,
    "InvertedResidualChannelsFused": InvertedResidualChannelsFused,
}


def get_active_fn(name):
    """Zero-arg activation factory by yml name (reference :461-469)."""
    return _ACTIVE_FNS[name]


def get_nl_norm_fn(name):
    """Normalisation class of the non-local block by yml name (reference :472-481)."""
    return _NL_NORMS[name]


def get_block(name):
    """Block class by yml name (reference :484-489)."""
    return _BLOCKS[name]


def _init_bn(m):
    if m.affine:
        (nn.init.zeros_ if isinstance(m, ZeroInitBN) else nn.init.ones_)(m.weight)
        nn.init.zeros_(m.bias)


def init_weights_slimmable(m):
    """Slimmable-network initialisation (reference :492-507)."""
    if isinstance(m, nn.Conv2d):
        nn.init.kaiming_normal_(m.weight, mode="fan_out")
        if m.bias is not None:
            nn.init.zeros_(m.bias)
    elif isinstance(m, nn.BatchNorm2d):
        _init_bn(m)
    elif isinstance(m, nn.Linear):
        nn.init.normal_(m.weight, 0, 0.01)
        nn.init.zeros_(m.bias)


def init_weights_mnas(m):
    """MnasNet initialisation (reference :510-537): conv ~ N(0, sqrt(2/fan_out)) with the
    depthwise fan_out = k*k, BN gamma=1 (0 for ZeroInitBN), Linear ~ U(+-1/sqrt(fan_out)).
    Consumes the RNG exactly like the reference so seeded models coincide."""
    if isinstance(m, nn.Conv2d):
        if m.groups == m.in_channels:
            fan_out = m.weight[0][0].numel()
        else:
            fan_out = nn.init._calculate_fan_in_and_fan_out(m.weight)[1]
        nn.init.normal_(m.weight, 0.0, nn.init.calculate_gain("relu") / math.sqrt(fan_out))
        if m.bias is not None:
            nn.init.zeros_(m.bias)
    elif isinstance(m, nn.BatchNorm2d):
        _init_bn(m)
    elif isinstance(m, nn.InstanceNorm2d):
        if m.affine:
            nn.init.zeros_(m.weight)
            nn.init.zeros_(m.bias)
    elif isinstance(m, nn.Linear):
        bound = 1.0 / math.sqrt(nn.init._calculate_fan_in_and_fan_out(m.weight)[1])
        nn.init.uniform_(m.weight, -bound, bound)
        nn.init.zeros_(m.bias)
