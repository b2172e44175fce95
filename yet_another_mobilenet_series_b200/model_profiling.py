"""Per-layer MACs, parameters and device time of a network of this package, with the surface and
the table of the reference's `utils/model_profiling.py`.

The reference counts through forward hooks on every module.  Here the blocks, the stem, the head
and the classifier launch kernels without calling their children, so no hook would fire.  Instead:

* MACs and parameters come from the input size propagated through the module tree, in the order
  the reference's forward calls the modules, with the reference's formula for each module kind.
  No kernel runs for them, so they are also counted with `use_cuda=False`.  The tree counted is
  the one the user sees: an AtomNAS hidden width of 23 counts as 23, not as the multiple of 8 the
  kernels run.
* The time column is the device time of the launches this package makes, not a host clock around
  torch modules re-run one by one.  `run_features` records a CUDA event at the boundary of each
  of its steps (`mobilenet_supernet.STEPS`): the stem, each block, the head, the pool and the
  classifier.  Each step's median over `num_forwards` forwards goes on the row of the module
  that step runs: the stem's and the head's convolution, the block, the pool, the classifier's
  Linear.  A block runs as one step (often one fused launch), so the rows of its children read 0.
"""
import logging
import statistics

import torch
from torch import nn

from . import mobilenet_base as mb
from . import mobilenet_supernet as sup
from .searched_network import MobileNetSearched

# the table's layout: a 95-character name column, then params, MACs and nanoseconds in 15 each
NAME_WIDTH = 95
COLUMN_WIDTH = 15
num_forwards = 10       # timed forwards per call, as many as the reference's `run_forward` makes

_ROW_KINDS = (nn.Conv2d, nn.Linear, nn.AvgPool2d, mb.SqueezeAndExcitation, mb.Nonlocal,
              mb.InvertedResidualChannels, mb.InvertedResidualChannelsFused)
_ABBREVIATIONS = (("kernel_size", "k"), ("stride", "s"), ("padding", "pad"), ("bias", "b"),
                  ("groups", "g"))


def conv_module_name_filter(name):
    """A module's repr with the convolution keywords abbreviated, as the table's names show it."""
    for word, short in _ABBREVIATIONS:
        name = name.replace(word, short)
    return name


def _line(name, *columns):
    return name.ljust(NAME_WIDTH) + "".join(c.rjust(COLUMN_WIDTH) for c in columns)


def _counts_line(name, m):
    return _line(name, "{:,}".format(m.n_params), "{:,}".format(m.n_macs),
                 "{:,}".format(m.n_seconds))


def _pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


def _window_out(size, k, s, pad, dil=(1, 1)):
    return tuple((n + 2 * p - d * (kk - 1) - 1) // ss + 1
                 for n, kk, ss, p, d in zip(size, k, s, pad, dil))


class _Counter:
    """Walks the module tree in the order the reference's forward calls it, from input shapes;
    sets n_macs / n_params / n_seconds (and `name` on a row) as the reference's hooks do."""

    def __init__(self, seconds):
        self.seconds = seconds      # {row module: ns}
        self.rows = []

    def _row(self, m, macs, params, name):
        m.n_macs, m.n_params, m.n_seconds, m.name = macs, params, self.seconds.get(m, 0), name
        self.rows.append(m)

    @staticmethod
    def _add(m, sub):
        m.n_macs += getattr(sub, "n_macs", 0)
        m.n_params += getattr(sub, "n_params", 0)
        m.n_seconds += getattr(sub, "n_seconds", 0)

    def visit(self, m, ins):
        """Output shape of `m` on an input of shape `ins`, after counting `m` and its callees."""
        if isinstance(m, nn.Conv2d):
            outs = (ins[0], m.out_channels) + _window_out(ins[2:], m.kernel_size, m.stride,
                                                          _pair(m.padding), m.dilation)
            self._row(m, (ins[1] * outs[1] * m.kernel_size[0] * m.kernel_size[1] * outs[2]
                          * outs[3] // m.groups) * outs[0], _params(m),
                      conv_module_name_filter(repr(m)))
            return outs
        if isinstance(m, nn.Linear):
            outs = (ins[0], m.out_features)
            self._row(m, ins[1] * outs[1] * outs[0], _params(m), repr(m))
            return outs
        if isinstance(m, nn.AvgPool2d):
            k = _pair(m.kernel_size)
            s = k if m.stride is None else _pair(m.stride)
            outs = tuple(ins[:2]) + _window_out(ins[2:], k, s, _pair(m.padding))
            # the reference's formula, exact when the stride equals the kernel size
            self._row(m, ins[1] * ins[2] * ins[3] * ins[0], 0, repr(m))
            return outs
        if isinstance(m, mb.SqueezeAndExcitation):
            pooled = (ins[0], ins[1], 1, 1)
            self.visit(m.se_expand, self.visit(m.active_fn, self.visit(m.se_reduce, pooled)))
            self._row(m, ins[1] * ins[2] * ins[3] * ins[0], 0, repr(m))
            self._add(m, m.se_reduce)
            self._add(m, m.se_expand)
            return ins
        if isinstance(m, mb.Nonlocal):
            self.visit(m.bn, self.visit(m.depthwise_conv, ins))
            n_in, H, W = ins[1], ins[2], ins[3]
            reduced_HW = (H // m.nl_s) * (W // m.nl_s)
            # the cost of the cheaper association order (a float: nl_c is a fraction)
            macs = min((H * W) * reduced_HW * n_in * (1 + m.nl_c),
                       (H * W) * n_in**2 * m.nl_c + reduced_HW * n_in**2 * m.nl_c)
            self._row(m, macs, 0, repr(m))
            self._add(m, m.depthwise_conv)
            return ins
        if isinstance(m, mb.InvertedResidualChannels):
            outs = [self.visit(op, ins) for op in m.ops][-1]
            self.visit(m.pw_bn, outs)
            self._row(m, 0, 0, repr(m))
            for op in m.ops:
                self._add(m, op)
            return outs
        if isinstance(m, mb.InvertedResidualChannelsFused):
            h = self.visit(m.expand_conv, ins)
            branches = [self.visit(op, h) for op in m.depth_ops]
            h = (branches[0][0], sum(b[1] for b in branches)) + tuple(branches[0][2:])
            outs = self.visit(m.nl_op, self.visit(m.project_conv, self.visit(m.se_op, h)))
            self._row(m, 0, 0, repr(m))
            for op in list(m.depth_ops) + [m.expand_conv, m.project_conv, m.se_op, m.nl_op]:
                self._add(m, op)
            return outs
        # the reference's generic branch: no row, the sums of the children it called
        if isinstance(m, nn.Sequential):
            outs = ins
            for child in m:
                outs = self.visit(child, outs)
        elif isinstance(m, (sup.MobileNetV2, MobileNetSearched)):
            # forward: features -> squeeze(3).squeeze(2) -> classifier
            outs = self.visit(m.classifier, self.visit(m.features, ins)[:2])
        elif isinstance(m, mb.Narrow):
            outs = tuple(m.length if d == m.dimension else n for d, n in enumerate(ins))
        elif next(m.children(), None) is None:
            outs = ins          # BatchNorm, activation, Dropout, Identity: shape kept
        else:
            raise NotImplementedError(
                "model_profiling cannot follow the forward of {}".format(type(m).__name__))
        m.n_macs, m.n_params, m.n_seconds = 0, 0, 0
        for child in m.children():
            self._add(m, child)
        return outs


def _params(m):
    return sum(p.numel() for p in m.parameters())


def _row_of(step_module):
    """The row a step's time goes on: the module's own, else the first row inside it (the stem's
    and the head's convolution, the classifier's Linear)."""
    return next(m for m in step_module.modules() if isinstance(m, _ROW_KINDS))


def _step_times(model, data):
    """{row module: median device ns of its run_features step} over `num_forwards` forwards."""
    runs = []
    for _ in range(num_forwards):
        sup.STEPS = marks = []
        try:
            model(data)
        finally:
            sup.STEPS = None
        torch.cuda.synchronize()
        runs.append([(m, e0.elapsed_time(e1)) for (_, e0), (m, e1) in zip(marks, marks[1:])])
    seconds = {}
    for i, (m, _) in enumerate(runs[0]):
        ms = statistics.median(run[i][1] for run in runs)
        seconds[_row_of(m)] = int(ms * 1e6)
    return seconds


def model_profiling(model, height, width, batch=1, channel=3, use_cuda=True, verbose=True):
    """Count (and with `use_cuda` time) every layer of `model` on a (batch, channel, height, width)
    input; returns (n_macs, n_params) of the whole model.

    Every module the reference's forward calls gets `n_macs`, `n_params` and `n_seconds`, and
    every row module a `name`.  With `verbose` the table is logged: one row per convolution,
    Linear, pool, Squeeze-and-Excitation, non-local block and block, then the Total.  With
    `use_cuda` the time column holds each row's median device time in ns (module docstring) on
    the model's CUDA device (a CPU model is moved to the current one and back); without, every
    time is 0 and nothing runs.  The model is left in eval mode."""
    model.eval()
    seconds = {}
    if use_cuda:
        origin = next(model.parameters()).device
        device = origin if origin.type == "cuda" else torch.device(
            "cuda", torch.cuda.current_device())
        model.to(device)
        # a generator of its own: the global RNG streams (dropout in training) stay untouched
        data = torch.rand(batch, channel, height, width, device=device,
                          generator=torch.Generator(device).manual_seed(0))
        with torch.cuda.device(device), torch.no_grad():
            model(data)                 # warm-up: plans, operand caches, module loads
            torch.cuda.synchronize()
            seconds = _step_times(model, data)
        model.to(origin)
    elif verbose:
        logging.info("model_profiling: the sm_90a path has no CPU timing; nanosecs are 0, "
                     "params and macs are counted from shapes.")
    counter = _Counter(seconds)
    counter.visit(model, (batch, channel, height, width))
    if verbose:
        rule = "-" * (NAME_WIDTH + 3 * COLUMN_WIDTH)
        logging.info(_line("Item", "params", "macs", "nanosecs"))
        logging.info(rule)
        for m in counter.rows:
            logging.info(_counts_line(m.name, m))
        logging.info(rule)
        logging.info(_counts_line("Total", model))
    return model.n_macs, model.n_params
