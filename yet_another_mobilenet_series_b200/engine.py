"""Host-side sequencing of the sm_90a kernels for one inverted-residual block.

A `BlockPlan` owns the HBM-resident intermediates of one block for one input shape
(NHWC bf16 [pixels, channels] matrices) and launches the kernels on them; `block_apply` is the
autograd entry the modules in `mobilenet_base.py` call.  Kernel order (train mode):

  forward   expand GEMM (+BN1 stats) -> depthwise (BN1+act on load, +BN2 stats)
            -> project GEMM (BN2+act operand transform, +BN3 stats) -> BN3 apply (+x)
  backward  BN3 reduce -> project dgrad GEMM (BN3-bwd operand transform, act'/BN2-bwd epilogue)
            + project wgrad GEMM -> depthwise bwd (BN2-bwd on load, fused wgrad, act'/BN1-bwd
            epilogue) -> expand dgrad GEMM (+dy) + expand wgrad GEMM, or both in one
            expand_bwd launch (expand_bwd_fused)

Reference semantics: models/mobilenet_base.py:446-451 (unfused), :330-342 (fused) and their
torch.autograd backward.  No tensor between the 1x1 convs is ever normalised in HBM: BatchNorm +
activation are applied by the consumer on load.
"""
import collections
import ctypes as C
import os

import torch

from . import native as nat

_ACT_CODE = {"none": 0, "relu": 1, "relu6": 2, "swish": 3, "hswish": 4}

# ---- instrumentation (bench.py / tests) ----------------------------------------------------------
# LAUNCHES counts every kernel launch made through the C ABI by this process.
# When PROFILE is a list, every launch is bracketed by CUDA events on the launching stream and
# (tag, algorithmic_bytes, flops, start_event, end_event) is appended.
LAUNCHES = 0
PROFILE = None


def launch(fn, st, tag="", nbytes=0, flops=0):
    """Enqueue one C-ABI kernel launch on torch's current stream."""
    global LAUNCHES
    LAUNCHES += 1
    if PROFILE is None:
        nat.check(fn(C.byref(st), nat.stream_handle()))
        return
    e0 = torch.cuda.Event(enable_timing=True)
    e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    nat.check(fn(C.byref(st), nat.stream_handle()))
    e1.record()
    PROFILE.append((tag, nbytes, flops, e0, e1))


def try_launch(fn, st, tag="", nbytes=0, flops=0):
    """`launch` for an entry point that may decline a shape: False, with nothing enqueued, when
    it returns YAMB_EINVAL (the caller then runs its unfused sequence); other errors raise."""
    global LAUNCHES
    e0 = None
    if PROFILE is not None:
        e0 = torch.cuda.Event(enable_timing=True)
        e0.record()
    rc = fn(C.byref(st), nat.stream_handle())
    if rc == nat.EINVAL:
        return False
    nat.check(rc)
    LAUNCHES += 1
    if PROFILE is not None:
        e1 = torch.cuda.Event(enable_timing=True)
        e1.record()
        PROFILE.append((tag, nbytes, flops, e0, e1))
    return True


# ---- weight-gradient side stream -------------------------------------------------------------------
# The split-K wgrad GEMMs feed nothing but the optimizer, so they leave the dgrad -> depthwise ->
# dgrad dependency chain: they are enqueued on a second stream right after the kernel that produces
# their last input and fill the SMs the chain's under-filled launches (7x7 / 14x14 layers: fewer
# tiles than SMs) and kernel tails leave idle.  `join_side()` makes the current stream wait for
# them.  With DEFER_JOIN False (default) every block joins at the end of its backward, so plain
# `loss.backward(); any_optimizer.step()` code is safe; TrainStep defers the join to the end of the
# whole backward.  YAMB_SIDE_WGRAD=0 puts everything back on one stream.
SIDE_WGRAD = os.environ.get("YAMB_SIDE_WGRAD", "1") != "0"
DEFER_JOIN = False
_side = {}


def _side_stream(dev):
    key = dev.index if dev.index is not None else torch.cuda.current_device()
    st = _side.get(key)
    if st is None:
        st = {"stream": torch.cuda.Stream(device=dev), "pending": False}
        _side[key] = st
    return st


def join_side(dev=None):
    """Current stream waits for every wgrad launched on the side stream so far."""
    for key, st in _side.items():
        if st["pending"] and (dev is None or key == (dev.index if dev.index is not None
                                                      else torch.cuda.current_device())):
            torch.cuda.current_stream().wait_stream(st["stream"])
            st["pending"] = False


def act_code_of(active_fn):
    """Activation code of the reference's zero-arg activation factory (get_active_fn)."""
    m = active_fn() if callable(active_fn) and not isinstance(active_fn, torch.nn.Module) \
        else active_fn
    name = type(m).__name__
    table = {"ReLU": 1, "ReLU6": 2, "Swish": 3, "HSwish": 4, "Identity": 0}
    if name not in table:
        raise ValueError("unsupported activation for the fused path: %s" % name)
    return table[name]


class Workspace:
    """Scratch of the statistics-producing kernels: the global accumulator of the per-channel sums
    (2*C doubles for a BatchNorm of C channels, room for C <= max_c; zero between launches — the
    last CTA of every launch returns it to zero) and the arrival counter.  The kernels of ONE
    stream serialise on it, so there is one per (device, stream): blocks driven from two streams at
    the same time (VERDICT r1) do not share."""
    _per_stream = {}

    def __init__(self, device):
        lib = nat.lib()
        self.max_ctas = lib.yamb_max_ctas()
        if self.max_ctas <= 0:
            raise nat.NativeError("no CUDA device visible to libyamb200 (there is no CPU path)")
        self.max_c = 4096
        # 2 * max_c doubles, kept in a float32 tensor
        self.partials = torch.zeros(4 * self.max_c, device=device, dtype=torch.float32)
        self.counter = torch.zeros(4, device=device, dtype=torch.int32)
        # slots 1 .. nat.DW_MAX_BRANCHES - 1: the branches of a grouped depthwise launch run at the
        # same time, each with its own accumulator (and counter[slot])
        self.branch_partials = torch.zeros((nat.DW_MAX_BRANCHES - 1) * 4 * self.max_c,
                                           device=device, dtype=torch.float32)
        self._se_sums = None
        self._se_sums_old = []

    def se_sums(self, n):
        """A float64 buffer of >= n elements for the per-(sample, channel) sums that pass from
        se_bwd_stats to se_bn_bwd_finalize within one block's backward (the kernels of one stream
        use it one block after the other).  A buffer that is outgrown stays alive: a captured CUDA
        graph may address it."""
        if self._se_sums is None or self._se_sums.numel() < n:
            if self._se_sums is not None:
                self._se_sums_old.append(self._se_sums)
            self._se_sums = torch.empty(n, device=self.partials.device, dtype=torch.float64)
        return self._se_sums

    def stats(self, C, slot=0):
        """(partials, counter) device pointers for a statistics kernel over C channels; `slot` > 0:
        those of branch `slot` of a grouped depthwise launch."""
        if C > self.max_c:
            raise nat.NativeError("BatchNorm of %d channels: the statistics accumulator holds %d"
                                  % (C, self.max_c))
        if slot == 0:
            return self.partials.data_ptr(), self.counter.data_ptr()
        return (self.branch_partials.data_ptr() + (slot - 1) * 4 * self.max_c * 4,
                self.counter.data_ptr() + 4 * slot)

    @classmethod
    def get(cls, device):
        idx = device.index if device.index is not None else torch.cuda.current_device()
        key = (idx, torch.cuda.current_stream(idx).cuda_stream)
        ws = cls._per_stream.get(key)
        if ws is None:
            ws = cls(device)
            cls._per_stream[key] = ws
        return ws


class Scratch:
    """Per-module kernel scratch (device buffers, C-ABI argument structs) cached in a module's
    `__dict__`.  It never travels with the module: a `copy.deepcopy` (the EMA model, reference
    common.py:164) or a pickle of the module gets None there and builds its own on first use
    (ctypes structs holding pointers can be neither copied nor pickled)."""

    def __deepcopy__(self, memo):
        return None

    def __reduce__(self):
        return (type(None), ())


class _ScratchDict(dict, Scratch):
    __deepcopy__ = Scratch.__deepcopy__
    __reduce__ = Scratch.__reduce__


def to_nhwc_bf16(x):
    """[N,C,H,W] any float dtype/layout -> channels_last bf16 (no copy if already so)."""
    if x.dtype != torch.bfloat16 or not x.is_contiguous(memory_format=torch.channels_last):
        x = x.to(dtype=torch.bfloat16, memory_format=torch.channels_last)
    return x


def _f32(n, dev):
    return torch.zeros(n, device=dev, dtype=torch.float32)


def _at(t, c0):
    """Device pointer of channel c0 of an fp32 per-channel tensor (None -> NULL)."""
    return None if t is None else t.data_ptr() + 4 * c0


class GradTargets:
    """Where the kernels of one backward accumulate the gradients of `params`, the parameters an
    autograd Function received, and what that Function returns for them.

    Direct mode: every parameter carries a pre-allocated `.grad` that the flat-arena optimizer
    marked `_yamb_direct`.  The kernels `+=` into those gradients and autograd gets None.
    Otherwise (autograd mode) the kernels accumulate into zeroed buffers made for this backward,
    which are returned to autograd as they are: nothing outlives the backward, so nothing needs a
    copy."""

    def __init__(self, params):
        self.params = list(params)
        self.direct = all(getattr(p, "_yamb_direct", False) and p.grad is not None
                          for p in self.params)
        self.grads = {}
        self.split = []      # (concatenated gradient, its parameters, dim): handed over by result()

    def of(self, p):
        """Accumulation target of `p`: its `.grad`, or a zeroed fp32 buffer of this backward."""
        if self.direct:
            return p.grad
        g = self.grads.get(id(p))
        if g is None:
            g = self.grads[id(p)] = torch.zeros(p.shape, device=p.device, dtype=torch.float32)
        return g

    def concat(self, params, dim, owner, key):
        """Accumulation target of 1x1 convolution weights concatenated along `dim` of their
        [out, in] matrices; one weight gets its own target.  In direct mode several weights share
        `owner[key]`, kept because a captured CUDA graph addresses it; in autograd mode a buffer
        of this backward.  Each weight gets its slice from `result()`."""
        if len(params) == 1:
            return self.of(params[0]).view(params[0].shape[:2])
        shape = list(params[0].shape[:2])
        shape[dim] = sum(p.shape[dim] for p in params)
        buf = owner.get(key) if self.direct else None
        if buf is None:
            buf = torch.zeros(shape, device=params[0].device, dtype=torch.float32)
            if self.direct:
                owner[key] = buf
        else:
            buf.zero_()
        self.split.append((buf, params, dim))
        return buf

    def put(self, p, g):
        """`g` is the finished gradient of `p` (added into `.grad` in direct mode)."""
        if self.direct:
            p.grad.add_(g)
        else:
            self.grads[id(p)] = g

    def put_all(self, params, grads):
        """`put` of a whole list: one multi-tensor add in direct mode."""
        if self.direct:
            torch._foreach_add_([p.grad for p in params], list(grads))
        else:
            self.grads.update((id(p), g) for p, g in zip(params, grads))

    @property
    def host_reads(self):
        """Whether anything on the current stream still reads what the kernels accumulated:
        autograd does in autograd mode, `result()` does to split a concatenated gradient."""
        return not self.direct or bool(self.split)

    def result(self):
        """The gradients autograd gets, in parameter order (None in direct mode and for the
        parameters without one)."""
        for buf, params, dim in self.split:
            c0 = 0
            for p in params:
                n = p.shape[dim]
                self.put(p, buf.narrow(dim, c0, n).reshape(p.shape))
                c0 += n
        if self.direct:
            return (None,) * len(self.params)
        return tuple(self.grads.get(id(p)) for p in self.params)


class _Bn:
    """Device-side state of one BatchNorm stage (possibly several reference BN modules whose
    channels are concatenated: per-branch BNs of the unfused block)."""

    def __init__(self, mods, dev):
        self.mods = list(mods)
        self.C = sum(m.num_features for m in self.mods)
        self.single = len(self.mods) == 1
        for name in ("scale", "shift", "mean", "invstd", "ca", "cb", "cc"):
            setattr(self, name, _f32(self.C, dev))
        self.dev = dev
        if not self.single:
            self.gamma = _f32(self.C, dev)
            self.beta = _f32(self.C, dev)
            self.dgamma = _f32(self.C, dev)
            self.dbeta = _f32(self.C, dev)
        self.eps = self.mods[0].eps
        self.slices = []
        c0 = 0
        for m in self.mods:
            self.slices.append((c0, m.num_features))
            c0 += m.num_features

    @property
    def batch_stats(self):
        m = self.mods[0]
        return m.training or not m.track_running_stats

    def momentum_value(self):
        m = self.mods[0].momentum
        return -1.0 if m is None else float(m)

    def gamma_beta(self):
        if self.single:
            return self.mods[0].weight, self.mods[0].bias
        torch.cat([m.weight.detach() for m in self.mods], out=self.gamma)
        torch.cat([m.bias.detach() for m in self.mods], out=self.beta)
        return self.gamma, self.beta

    def eval_coeffs(self):
        """scale/shift from running statistics (eval mode)."""
        rm = torch.cat([m.running_mean for m in self.mods]) if not self.single \
            else self.mods[0].running_mean
        rv = torch.cat([m.running_var for m in self.mods]) if not self.single \
            else self.mods[0].running_var
        g, b = self.gamma_beta()
        torch.rsqrt(rv + self.eps, out=self.invstd)
        torch.mul(g.detach(), self.invstd, out=self.scale)
        self.mean.copy_(rm)
        torch.addcmul(b.detach(), rm, self.scale, value=-1.0, out=self.shift)

    def _module(self, c0, C):
        """(index, channel offset) of the reference module that holds channels [c0, c0+C): any
        range of a single module, exactly one module's channels otherwise."""
        if self.single:
            return 0, c0
        for i, (s0, n) in enumerate(self.slices):
            if (s0, n) == (c0, C):
                return i, 0
        raise nat.NativeError("BatchNorm slice does not match a reference module")

    def fwd_struct(self, count, c0=0, C=None, slot=0):
        """yamb_bn_fwd of channels [c0, c0+C) (all by default) over `count` rows, with the
        statistics workspace of the current stream (its `slot`, see Workspace.stats): build it
        right before its launch."""
        C = self.C if C is None else C
        i, off = self._module(c0, C)
        m = self.mods[i]
        s = nat.BnFwd()
        s.partials, s.counter = Workspace.get(self.dev).stats(C, slot)
        s.gamma, s.beta = _at(m.weight, off), _at(m.bias, off)
        s.eps, s.momentum = self.eps, self.momentum_value()
        if m.track_running_stats and m.running_mean is not None:
            s.running_mean, s.running_var = _at(m.running_mean, off), _at(m.running_var, off)
            s.num_batches_tracked = nat.ptr(m.num_batches_tracked)
        s.scale, s.shift = _at(self.scale, c0), _at(self.shift, c0)
        s.mean, s.invstd = _at(self.mean, c0), _at(self.invstd, c0)
        s.count = count
        return s

    def bwd_struct(self, count, grads, c0=0, C=None, slot=0):
        """yamb_bn_bwd of channels [c0, c0+C) (all by default) over `count` rows; grads: the
        (dgamma, dbeta) accumulation targets of every module.  Built like `fwd_struct`."""
        C = self.C if C is None else C
        i, off = self._module(c0, C)
        s = nat.BnBwd()
        s.partials, s.counter = Workspace.get(self.dev).stats(C, slot)
        s.gamma = _at(self.mods[i].weight, off)
        s.mean, s.invstd = _at(self.mean, c0), _at(self.invstd, c0)
        dg, db = grads[i]
        s.dgamma, s.dbeta = _at(dg, off), _at(db, off)
        s.ca, s.cb, s.cc = _at(self.ca, c0), _at(self.cb, c0), _at(self.cc, c0)
        s.count = count
        s.use_batch_stats = 1 if self.batch_stats else 0
        return s


BlockParts = collections.namedtuple(
    "BlockParts", "fused expand_convs bn1s dws project_convs bn3 se nl")


def _present(op):
    """The SE / non-local child, or None where the reference placed its Identity placeholder."""
    return None if type(op).__name__ == "Identity" else op


def block_parts(block):
    """The child modules of either block class (reference models/mobilenet_base.py:206-458):
    expand convs and BN1s (one per branch for InvertedResidualChannels, one for
    InvertedResidualChannelsFused, none without the expansion), (conv, BN2) of every branch's
    depthwise stage, the project convs, BN3, the Squeeze-and-Excitation and non-local modules (None
    when absent; always None for the unfused class)."""
    if hasattr(block, "expand_conv"):
        dws = [list(op.children())[-1] for op in block.depth_ops]
        exp = [block.expand_conv] if block.expand else []
        return BlockParts(True, [e[0] for e in exp], [e[1] for e in exp],
                          [(d[0], d[1]) for d in dws], [block.project_conv[0]],
                          block.project_conv[1], _present(block.se_op), _present(block.nl_op))
    exp = [op[0] for op in block.ops] if block.expand else []
    first = 1 if block.expand else 0       # ops[i] = [ConvBNReLU expand], ConvBNReLU dw, Conv2d
    return BlockParts(False, [e[0] for e in exp], [e[1] for e in exp],
                      [(op[first][0], op[first][1]) for op in block.ops],
                      [op[first + 1] for op in block.ops], block.pw_bn, None, None)


def _nl_norm_supported(norm):
    """The non-local block's norms the sm_90a path runs (reference get_nl_norm_fn,
    models/mobilenet_base.py:472-481): BatchNorm2d (`nl_norm: nn.BatchNorm`, the default) and the
    tracked affine InstanceNorm2d (`nl_norm: nn.InstanceNorm`)."""
    if isinstance(norm, torch.nn.BatchNorm2d):
        return True
    return isinstance(norm, torch.nn.InstanceNorm2d) and norm.affine and \
        norm.track_running_stats and norm.running_mean is not None


# ---- kernel calls made from several places -------------------------------------------------------
# Activations are bf16 [pixels, C] matrices, per-channel vectors fp32; one branch of a wider
# activation is a column slice (a view), so C and the row pitch come from the tensor.  `stats` is
# a yamb_bn_fwd / yamb_bn_bwd struct from `_Bn.fwd_struct` / `bwd_struct`, built by the caller
# right before the call.

def _bn_apply(bn, h, y, act, tag, residual=None, residual2=None):
    """y = act(scale*h + shift) (+ residual) (+ residual2) with the coefficients of `bn` (a
    `_Bn`); dense [M, C] operands."""
    M, Cc = h.shape
    a = nat.BnApply()
    a.M, a.C, a.ldh, a.ldr, a.ldy = M, Cc, Cc, Cc, Cc
    a.h, a.scale, a.shift, a.act = h.data_ptr(), bn.scale.data_ptr(), bn.shift.data_ptr(), act
    a.residual, a.y = nat.ptr(residual), y.data_ptr()
    if residual2 is not None:
        a.residual2, a.ldr2 = residual2.data_ptr(), Cc
    operands = 2 + (residual is not None) + (residual2 is not None)
    launch(nat.lib().yamb_bn_apply_fwd, a, tag, 2 * M * Cc * operands)


def _bn_reduce(stats, dy, h, tag, z=None):
    """BatchNorm backward statistics of dy over dense [M, C] dy and h, finalised by `stats`;
    z = (z_scale, z_shift, act): dy is first multiplied by act'(z_scale*h + z_shift)."""
    M, Cc = h.shape
    r = nat.BnReduce()
    r.M, r.C, r.lddy, r.ldh = M, Cc, Cc, Cc
    r.dy, r.h, r.bn = dy.data_ptr(), h.data_ptr(), C.pointer(stats)
    if z is not None:
        r.z_scale, r.z_shift, r.z_act = z
    launch(nat.lib().yamb_bn_reduce_bwd, r, tag, 4 * M * Cc)


def _bn_bwd_apply(bn, dy, h, dh, tag, z=None):
    """dh = ca*dy + cb*h + cc with the backward coefficients of `bn` (a `_Bn`), dy taken as in
    `_bn_reduce`; dense [M, C] operands."""
    M, Cc = h.shape
    a = nat.BnBwdApply()
    a.M, a.C, a.lddy, a.ldh, a.lddh = M, Cc, Cc, Cc, Cc
    a.dy, a.h, a.dh = dy.data_ptr(), h.data_ptr(), dh.data_ptr()
    if z is not None:
        a.z_scale, a.z_shift, a.z_act = z
    a.ca, a.cb, a.cc = bn.ca.data_ptr(), bn.cb.data_ptr(), bn.cc.data_ptr()
    launch(nat.lib().yamb_bn_bwd_apply_bwd, a, tag, 6 * M * Cc)


def _dw_fwd(conv, nhw, x, y, tag, pre=None, stats=None):
    """y = depthwise `conv` of x over N x H x W pixels (x read with y's pitch); pre = (scale,
    shift, act) is applied to x on load; `stats` takes y's BatchNorm statistics."""
    d, nbytes, flops = _dw_fwd_args(conv, nhw, x, y, pre, stats)
    launch(nat.lib().yamb_depthwise_fwd, d, tag, nbytes, flops)


def _dw_fwd_args(conv, nhw, x, y, pre=None, stats=None):
    """(yamb_dw_fwd, bytes, flops) of `_dw_fwd`."""
    k, s = conv.kernel_size[0], conv.stride[0]
    Cc = y.shape[1]
    d = nat.DwFwd()
    N, H, W = d.N, d.H, d.W = nhw
    d.C, d.ldc, d.k, d.stride = Cc, y.stride(0), k, s
    d.x, d.w, d.y = x.data_ptr(), conv.weight.data_ptr(), y.data_ptr()
    if pre is not None:
        d.in_scale, d.in_shift, d.in_act = pre[0].data_ptr(), pre[1].data_ptr(), pre[2]
    if stats is not None:
        d.bn = C.pointer(stats)
    m_in, m_out = N * H * W, N * ((H - 1) // s + 1) * ((W - 1) // s + 1)
    return d, 2 * Cc * (m_in + m_out), 2 * m_out * Cc * k * k


def _dw_bwd(conv, nhw, dz, h, coef, dw, x, dx, tag, pre=None, residual=None, stats=None, se=None):
    """Backward of `_dw_fwd` from the output gradient ca*dz + cb*h + cc (coef = (ca, cb, cc)):
    weight gradient += into dw, input gradient into dx, taken back through `pre` when given (its
    BatchNorm backward statistics into `stats`), + residual.  Every matrix is read with dz's
    pitch.  se = (gate, dpool, scale, shift, act) of a Squeeze-and-Excitation block: dz is then
    dY = d(a2*gate) and the kernel forms dz2 = (dY*gate + dpool)*act'(scale*h + shift) on load
    (yamb_depthwise_bwd_se)."""
    d, nbytes, flops = _dw_bwd_args(conv, nhw, dz, h, coef, dw, x, dx, pre, residual, stats)
    if se is None:
        launch(nat.lib().yamb_depthwise_bwd, d, tag, nbytes, flops)
        return
    a = nat.DwBwdSe()
    a.dw = d
    a.gate, a.dpool, a.ldg = se[0].data_ptr(), se[1].data_ptr(), se[0].stride(0)
    a.scale, a.shift, a.act = se[2].data_ptr(), se[3].data_ptr(), se[4]
    launch(nat.lib().yamb_depthwise_bwd_se, a, tag + "_se", nbytes, flops)


def _dw_bwd_args(conv, nhw, dz, h, coef, dw, x, dx, pre=None, residual=None, stats=None):
    """(yamb_dw_bwd, bytes, flops) of `_dw_bwd` without `se`."""
    k, s = conv.kernel_size[0], conv.stride[0]
    Cc = dz.shape[1]
    d = nat.DwBwd()
    N, H, W = d.N, d.H, d.W = nhw
    d.C, d.ldc, d.k, d.stride = Cc, dz.stride(0), k, s
    d.dz, d.h = dz.data_ptr(), h.data_ptr()
    d.ca, d.cb, d.cc = (t.data_ptr() for t in coef)
    d.w, d.dw = conv.weight.data_ptr(), dw.data_ptr()
    d.x, d.dx, d.residual = x.data_ptr(), dx.data_ptr(), nat.ptr(residual)
    if pre is not None:
        d.in_scale, d.in_shift, d.in_act = pre[0].data_ptr(), pre[1].data_ptr(), pre[2]
    if stats is not None:
        d.bn = C.pointer(stats)
    m_in, m_out = N * H * W, N * ((H - 1) // s + 1) * ((W - 1) // s + 1)
    return d, 4 * Cc * (m_in + m_out), 4 * m_out * Cc * k * k


def _se_fc(se, pooled, u, v, gate, packed=None):
    """gate = sigmoid(W_e act(W_r pooled + b_r) + b_e) of the Squeeze-and-Excitation module `se`
    on pooled [N, C], keeping u = W_r pooled + b_r and v = act(u) [N, R] (fp32 throughout).
    packed: (W_r, W_e, b_e) over another hidden order (the multi-branch eval path) instead of the
    module's own."""
    N, Cc = pooled.shape
    R = se.se_reduce.weight.shape[0]
    w_r, w_e, b_e = packed or (se.se_reduce.weight, se.se_expand.weight, se.se_expand.bias)
    f = nat.SeFc()
    f.N, f.C, f.R, f.act = N, Cc, R, act_code_of(se.active_fn)
    f.pooled = pooled.data_ptr()
    f.w_r, f.b_r = w_r.data_ptr(), se.se_reduce.bias.data_ptr()
    f.w_e, f.b_e = w_e.data_ptr(), b_e.data_ptr()
    f.u, f.v, f.gate = u.data_ptr(), v.data_ptr(), gate.data_ptr()
    launch(nat.lib().yamb_se_fc_fwd, f, "se_fc", 4 * N * Cc * 2, 4 * N * Cc * R)


class _NlTail:
    """Non-local block (reference models/mobilenet_base.py:158-173) behind a BatchNorm output l,
    for one shape: y = norm(dw3x3(f)) + l (+ x), f = (W/H) theta (phi^T g).  Owns l, f, h (bf16
    [N*H*W, C]) and F (fp32 [N][c][C]); `forward` is the four launches of the training plan and of
    the eval path alike, `backward` the training plan's way back to dl (its buffers are made on
    the first backward: the eval path never needs them).

    The norm (`bn4`) runs in one of three modes, chosen per forward: BatchNorm with batch
    statistics (the depthwise kernel takes them, yamb_bn_apply_fwd applies them), InstanceNorm with
    per-sample statistics (yamb_instance_norm_fwd takes and applies them), or either norm folded
    from its running statistics (yamb_bn_apply_fwd)."""

    def __init__(self, nl, bn4, N, H, W, C, dev):
        self.nl, self.bn4 = nl, bn4
        self.instance = isinstance(nl.bn, torch.nn.InstanceNorm2d)
        self.used_instance_stats = False      # mode of the last forward (its backward follows it)
        self.in_mean = self.in_invstd = None
        self.N, self.H, self.W, self.C, self.M = N, H, W, C, N * H * W
        self.cr = int(nl.nl_c * C)             # theta / phi channels (:163)
        self.sub = int(nl.nl_s)
        if self.cr <= 0 or self.cr % 2 or self.sub < 1:
            raise nat.NativeError("non-local block: int(nl_c * C) must be a positive even "
                                  "number (got %d)" % self.cr)
        self.scale = float(W) / float(H)       # sic `f / H * W` (:171)
        bf = torch.bfloat16
        self.l = torch.empty(self.M, C, device=dev, dtype=bf)
        self.f = torch.empty(self.M, C, device=dev, dtype=bf)
        self.h = torch.empty(self.M, C, device=dev, dtype=bf)
        self.F = _f32(N * self.cr * C, dev)
        self.df = self.dl = self.dF = None
        self.in_dh = None

    def gram(self, X, I, Y, sub, alpha, G, tag):
        g = nat.NlGram()
        g.N, g.H, g.W, g.sub = self.N, self.H, self.W, sub
        g.X, g.ldx, g.I = X.data_ptr(), self.C, I
        g.Y, g.ldy, g.J = Y.data_ptr(), self.C, self.C
        g.alpha, g.G = alpha, G.data_ptr()
        launch(nat.lib().yamb_nl_gram_fwd, g, tag, 4 * self.M * self.C // (sub * sub))

    def rowmat(self, X, K, Mat, sk, so, O, sub, alpha, out, tag, base=None, accumulate=0):
        r = nat.NlRowmat()
        r.N, r.H, r.W, r.sub = self.N, self.H, self.W, sub
        r.X, r.ldx, r.K = X.data_ptr(), self.C, K
        r.Mat, r.mat_stride, r.sk, r.so, r.O = Mat.data_ptr(), self.cr * self.C, sk, so, O
        r.alpha = alpha
        if base is not None:
            r.base, r.ldb, r.O_copy = base.data_ptr(), self.C, self.C
        r.accumulate = accumulate
        r.out, r.ldo = out.data_ptr(), self.C
        launch(nat.lib().yamb_nl_rowmat_fwd, r, tag, 4 * self.M * self.C // (sub * sub))

    def forward(self, xm, y, residual):
        """self.l -> y."""
        Cc, c = self.C, self.cr
        instance = self.instance and self.bn4.batch_stats
        if instance and self.H * self.W == 1:
            raise nat.NativeError("non-local block: InstanceNorm in training mode needs more than "
                                  "one pixel per channel (the map is 1x1)")
        self.used_instance_stats = instance
        # F = phi^T g over the sub-sampled pixels; f = (W/H) theta F
        self.gram(self.l, c, self.l, self.sub, 1.0, self.F, "nl_gram")
        self.rowmat(self.l, c, self.F, Cc, 1, Cc, 1, self.scale, self.f, "nl_apply")
        # depthwise 3x3 (no activation before it) + BN4 statistics (InstanceNorm: per sample, by
        # yamb_instance_norm_fwd)
        if not self.bn4.batch_stats:
            self.bn4.eval_coeffs()
        _dw_fwd(self.nl.depthwise_conv, (self.N, self.H, self.W), self.f, self.h, "nl_dw_fwd",
                stats=self.bn4.fwd_struct(self.M) if self.bn4.batch_stats and not instance
                else None)
        if instance:
            self._instance_forward(xm, y, residual)
            return
        # y = BN4(h) + l (+ x)
        _bn_apply(self.bn4, self.h, y, 0, "nl_bn_apply", residual=self.l,
                  residual2=xm if residual else None)

    def _instance_forward(self, xm, y, residual):
        """y = InstanceNorm(h) + l (+ x) with per-sample statistics; mean / invstd [N][C] kept for
        the backward, running statistics updated (torch: momentum None -> no update)."""
        Cc = self.C
        m = self.bn4.mods[0]
        if self.in_mean is None:
            self.in_mean = _f32(self.N * Cc, self.l.device)
            self.in_invstd = _f32(self.N * Cc, self.l.device)
        s = nat.InFwd()
        s.N, s.HW, s.C, s.ldh = self.N, self.H * self.W, Cc, Cc
        s.h = self.h.data_ptr()
        s.gamma, s.beta = m.weight.data_ptr(), m.bias.data_ptr()
        s.eps = m.eps
        s.momentum = 0.0 if m.momentum is None else float(m.momentum)
        s.running_mean, s.running_var = m.running_mean.data_ptr(), m.running_var.data_ptr()
        s.mean, s.invstd = self.in_mean.data_ptr(), self.in_invstd.data_ptr()
        s.residual, s.ldr = self.l.data_ptr(), Cc
        if residual:
            s.residual2, s.ldr2 = xm.data_ptr(), Cc
        s.y, s.ldy = y.data_ptr(), Cc
        s.counter = Workspace.get(self.l.device).counter.data_ptr()
        launch(nat.lib().yamb_instance_norm_fwd, s, "nl_in_fwd",
               2 * self.M * Cc * (5 if residual else 4))

    def instance_backward(self, dym, dh, grads):
        """dh = InstanceNorm backward of dy (bf16), dgamma / dbeta += into grads[0]."""
        Cc = self.C
        m = self.bn4.mods[0]
        s = nat.InBwd()
        s.N, s.HW, s.C = self.N, self.H * self.W, Cc
        s.ldh = s.lddy = s.lddh = Cc
        s.dy, s.h = dym.data_ptr(), self.h.data_ptr()
        s.gamma = m.weight.data_ptr()
        s.mean, s.invstd = self.in_mean.data_ptr(), self.in_invstd.data_ptr()
        dg, db = grads[0]
        s.dgamma, s.dbeta = nat.ptr(dg), nat.ptr(db)
        s.dh = dh.data_ptr()
        s.counter = Workspace.get(self.l.device).counter.data_ptr()
        launch(nat.lib().yamb_instance_norm_bwd, s, "nl_in_bwd", 2 * self.M * Cc * 5)

    def backward(self, dym, grads):
        """dy -> dl (gradient of the BN3 output): norm backward, depthwise 3x3 backward, the two
        products' backward, plus the `+ l` pass-through.  grads: the plan's accumulation targets
        ('bn4', 'nl_dw')."""
        Cc, c, bf, dev = self.C, self.cr, torch.bfloat16, self.l.device
        if self.df is None:
            self.df = torch.empty(self.M, Cc, device=dev, dtype=bf)
            self.dl = torch.empty(self.M, Cc, device=dev, dtype=bf)
            self.dF = _f32(self.N * c * Cc, dev)
        if self.used_instance_stats:
            # InstanceNorm with per-sample statistics: its backward writes dh (bf16), which the
            # depthwise backward takes with the identity coefficients ca = 1, cb = cc = 0
            if self.in_dh is None:
                self.in_dh = torch.empty(self.M, Cc, device=dev, dtype=bf)
                self.ones = torch.ones(Cc, device=dev, dtype=torch.float32)
                self.zeros = _f32(Cc, dev)
            self.instance_backward(dym, self.in_dh, grads["bn4"])
            dz, coef = self.in_dh, (self.ones, self.zeros, self.zeros)
        else:
            _bn_reduce(self.bn4.bwd_struct(self.M, grads["bn4"]), dym, self.h, "nl_bn_reduce")
            dz, coef = dym, (self.bn4.ca, self.bn4.cb, self.bn4.cc)
        _dw_bwd(self.nl.depthwise_conv, (self.N, self.H, self.W), dz, self.h, coef,
                grads["nl_dw"], self.f, self.df, "nl_dw_bwd")
        # dF = (W/H) theta^T df (all pixels);  dl = dy + [dtheta | 0];  sub-sampled rows += dphi, dg
        self.gram(self.l, c, self.df, 1, self.scale, self.dF, "nl_gram_bwd")
        self.rowmat(self.df, Cc, self.F, 1, Cc, c, 1, self.scale, self.dl, "nl_dtheta", base=dym)
        self.rowmat(self.l, Cc, self.dF, 1, Cc, c, self.sub, 1.0, self.dl, "nl_dphi", accumulate=1)
        self.rowmat(self.l, c, self.dF, Cc, 1, Cc, self.sub, 1.0, self.dl, "nl_dg", accumulate=1)
        return self.dl


class BlockPlan:
    """The training-path kernel sequence of one block for one input shape, with the HBM-resident
    intermediates it owns.  Every C-ABI argument struct is built per call, right before its
    launch: a BatchNorm struct carries the statistics workspace of the stream it is launched on
    (`Workspace.get`), and the same plan may run on another stream next time."""

    def __init__(self, block, x):
        dev = x.device
        self.dev = dev
        N, Cin, H, W = x.shape
        self.N, self.H, self.W, self.Cin = N, H, W, Cin
        self.stride = block.stride
        # pad=(k-1)//2, odd k: out = floor((H-1)/s)+1
        self.Ho = (H - 1) // self.stride + 1
        self.Wo = (W - 1) // self.stride + 1
        self.Cout = block.output_dim
        self.channels = list(block.channels)
        self.expand = bool(block.expand)
        self.residual = bool(block.use_res_connect)
        self.act = act_code_of(block.active_fn)
        parts = block_parts(block)
        self.fused = parts.fused
        self.Chid = sum(self.channels)
        if self.Cin % 8 or self.Cout % 8 or any(c % 8 for c in self.channels):
            raise nat.NativeError(
                "channel counts must be multiples of 8 for the sm_90a path "
                "(inp=%d oup=%d hidden=%s)" % (self.Cin, self.Cout, self.channels))
        if not self.expand and not self.fused and len(self.channels) > 1:
            raise nat.NativeError("expand=False with several branches is not supported")
        self.M_in = N * H * W
        self.M_out = N * self.Ho * self.Wo
        bf = torch.bfloat16
        Chid, Cout = self.Chid, self.Cout
        # ---- intermediates (raw, pre-BatchNorm) ----
        self.h1 = torch.empty(self.M_in, Chid, device=dev, dtype=bf) if self.expand else None
        self.h2 = torch.empty(self.M_out, Chid, device=dev, dtype=bf)
        self.h3 = torch.empty(self.M_out, Cout, device=dev, dtype=bf)
        self.dh3 = None
        self.dz2 = None
        self.dz1 = None
        # ---- modules ----
        self.conv_exp, self.conv_proj = parts.expand_convs, parts.project_convs
        self.se, self.nl = parts.se, parts.nl
        if self.nl is not None:
            # non-local block (reference models/mobilenet_base.py:131-178) between BN3 and the skip
            nl = self.nl
            if not _nl_norm_supported(nl.bn):
                raise nat.NativeError(
                    "non-local block: the sm_90a path runs nn.BatchNorm2d and "
                    "nn.InstanceNorm2d(affine=True, track_running_stats=True) as nl_norm (got %r)"
                    % nl.bn)
            self.nl_tail = _NlTail(nl, _Bn([nl.bn], dev), N, self.Ho, self.Wo, Cout, dev)
            self.bn4 = self.nl_tail.bn4
        if self.se is not None:
            self.se_act = act_code_of(self.se.active_fn)
            self.se_r = self.se.se_reduce.weight.shape[0]
            self.se_u = _f32(N * self.se_r, dev).view(N, self.se_r)
            self.se_v = _f32(N * self.se_r, dev).view(N, self.se_r)
            self.se_du = _f32(N * self.se_r, dev).view(N, self.se_r)
            self.se_dt = _f32(N * Chid, dev).view(N, Chid)
            self.pooled = _f32(N * Chid, dev).view(N, Chid)
            self.gate = _f32(N * Chid, dev).view(N, Chid)
            self.dgate = _f32(N * Chid, dev).view(N, Chid)
            self.dpool = _f32(N * Chid, dev).view(N, Chid)
        self.conv_dw = [conv for conv, _ in parts.dws]
        self.expand_dw_kind = expand_dw_kind(block, H, W)
        self.mb_dw_kind = mb_dw_kind(block, H, W)
        self.bn1 = _Bn(parts.bn1s, dev) if self.expand else None
        self.bn2 = _Bn([bn for _, bn in parts.dws], dev)
        self.bn3 = _Bn([parts.bn3], dev)
        # ---- bf16 tensor-core operands ----
        self.w_exp_bf = torch.empty(Chid, Cin, device=dev, dtype=bf) if self.expand else None
        self.w_proj_bf = torch.empty(Cout, Chid, device=dev, dtype=bf)
        self.w_exp_own, self.w_proj_own = self.w_exp_bf, self.w_proj_bf
        # backward: the expand-side gradients in one yamb_expand_bwd launch, or two GEMMs
        self.expand_fused = self.expand and expand_bwd_fused(self.M_in, Cin, Chid)
        # multi-branch expand / project weight gradients of direct mode (GradTargets.concat)
        self.concat_grads = {}
        self.generation = 0
        self.pinned = False

    # -- helpers -------------------------------------------------------------------------------
    def _refresh_weights(self):
        """fp32 master -> bf16 tensor-core operands (merged over branches).

        A single-branch weight uses the fused optimizer's bf16 mirror arena directly.  The mirror
        is rewritten by `yamb_rmsprop_step` (a raw-pointer write that does not touch the tensor's
        version counter); any OTHER in-place write to the fp32 master (load_state_dict, a DDP
        broadcast, re-initialisation, an EMA swap-in) bumps `_version`, which is detected here and
        the mirror is re-cast before use."""
        with torch.no_grad():
            if self.expand:
                if len(self.conv_exp) == 1:
                    self.w_exp_bf = _bf16_operand(self.conv_exp[0].weight, self.w_exp_own,
                                                  (self.Chid, self.Cin))
                else:
                    self.w_exp_bf.copy_(torch.cat([c.weight.flatten(1) for c in self.conv_exp]))
            if len(self.conv_proj) == 1:
                self.w_proj_bf = _bf16_operand(self.conv_proj[0].weight, self.w_proj_own,
                                               (self.Cout, self.Chid))
            else:
                self.w_proj_bf.copy_(torch.cat([c.weight.flatten(1) for c in self.conv_proj], 1))

    def _fork_event(self):
        if not SIDE_WGRAD or PROFILE is not None:
            return None
        ev = torch.cuda.Event()
        ev.record()
        return ev

    def _call_side(self, fn, st, tag, nbytes, flops, ev, tensors):
        """Launch on the wgrad side stream once `ev` (recorded on the main stream) has passed."""
        if ev is None:
            return launch(fn, st, tag, nbytes, flops)
        side = _side_stream(self.dev)
        side["stream"].wait_event(ev)
        with torch.cuda.stream(side["stream"]):
            launch(fn, st, tag, nbytes, flops)
        for t in tensors:    # caller-owned storage read by the side stream: keep it alive for it
            t.record_stream(side["stream"])
        side["pending"] = True

    # -- forward ---------------------------------------------------------------------------------
    def forward(self, x, pre=None):
        """x: channels_last bf16 [N,Cin,H,W]; returns channels_last bf16 [N,Cout,Ho,Wo].
        pre = (scale, shift, act) of an input BatchNorm + activation (a block without expansion
        whose x is the raw output of the layer before): the depthwise applies it to x on load."""
        lib = nat.lib()
        self.generation += 1
        self._refresh_weights()
        xm = x.permute(0, 2, 3, 1).reshape(self.M_in, self.Cin)  # view, NHWC matrix
        y = torch.empty((self.N, self.Cout, self.Ho, self.Wo), device=self.dev,
                        dtype=torch.bfloat16, memory_format=torch.channels_last)
        # 1. expand 1x1 + BN1 statistics: the GEMM finalises the statistics of one BatchNorm
        #    module, so with one module per branch it runs once per branch slice
        if self.expand:
            stats = self.bn1.batch_stats
            if not stats:
                self.bn1.eval_coeffs()
            for c0, cb in self.bn1.slices if stats else [(0, self.Chid)]:
                s = slice(c0, c0 + cb)
                g = nat.Gemm()
                g.M, g.N, g.K = self.M_in, cb, self.Cin
                g.A, g.lda = xm.data_ptr(), self.Cin
                g.B, g.ldb = self.w_exp_bf[s].data_ptr(), self.Cin
                g.D, g.ldd = self.h1[:, s].data_ptr(), self.Chid
                if stats:
                    g.bn_fwd = C.pointer(self.bn1.fwd_struct(self.M_in, c0, cb))
                launch(lib.yamb_pointwise_gemm, g, "pw_expand_fwd",
                       2 * self.M_in * (self.Cin + cb), 2 * self.M_in * self.Cin * cb)
        # 2. depthwise per branch (BN1+act applied on load) + BN2 statistics; without the
        #    expansion hidden == inp, so x has the hidden pitch.  TRAIN_EXPAND_DW_FUSED: the
        #    expanded tile recomputed from x instead of reading h1 back, where the kernel covers it
        if not self.bn2.batch_stats:
            self.bn2.eval_coeffs()
        if not (expand_dw_fused(self) and self._expand_dw_train(xm)) and \
                not (mb_dw_grouped(self) and self._dw_fwd_grouped()):
            for (c0, cb), conv in zip(self.bn2.slices, self.conv_dw):
                s = slice(c0, c0 + cb)
                _dw_fwd(conv, (self.N, self.H, self.W), self.h1[:, s] if self.expand else xm,
                        self.h2[:, s], "dw_fwd",
                        pre=(self.bn1.scale[s], self.bn1.shift[s], self.act) if self.expand
                        else pre,
                        stats=self.bn2.fwd_struct(self.M_out, c0, cb) if self.bn2.batch_stats
                        else None)
        # 2b. Squeeze-and-Excitation gate (reference mobilenet_base.py:110-113): spatial mean of
        #     a2 = act(bn2(h2)) by a kernel, the two fully connected layers + sigmoid by another,
        #     the gate applied inside the project GEMM's operand transform
        if self.se is not None:
            sp = nat.SePool()
            sp.N, sp.HW, sp.C, sp.ldh = self.N, self.Ho * self.Wo, self.Chid, self.Chid
            sp.h, sp.scale, sp.shift, sp.act = self.h2.data_ptr(), self.bn2.scale.data_ptr(), \
                self.bn2.shift.data_ptr(), self.act
            sp.pooled = self.pooled.data_ptr()
            launch(lib.yamb_se_pool_fwd, sp, "se_pool", 2 * self.M_out * self.Chid)
            # the two fully connected layers on the pooled [N, C] vectors (fp32, like the reference
            # keeps them) + sigmoid: one launch (csrc/se_fc.cu)
            _se_fc(self.se, self.pooled, self.se_u, self.se_v, self.gate)
        # 3. project 1x1 (BN2+act as operand transform) + BN3 statistics
        g = nat.Gemm()
        g.M, g.N, g.K = self.M_out, self.Cout, self.Chid
        g.A, g.lda = self.h2.data_ptr(), self.Chid
        g.B, g.ldb = self.w_proj_bf.data_ptr(), self.Chid
        g.D, g.ldd = self.h3.data_ptr(), self.Cout
        g.a_xform, g.a_act = 1, self.act
        g.a_scale, g.a_shift = self.bn2.scale.data_ptr(), self.bn2.shift.data_ptr()
        if self.se is not None:
            g.a_gate, g.gate_rows_per_sample = self.gate.data_ptr(), self.Ho * self.Wo
        if self.bn3.batch_stats:
            g.bn_fwd = C.pointer(self.bn3.fwd_struct(self.M_out))
        else:
            self.bn3.eval_coeffs()
        launch(lib.yamb_pointwise_gemm, g, "pw_project_fwd",
               2 * self.M_out * (self.Chid + self.Cout),
               2 * self.M_out * self.Chid * self.Cout)
        # 4. BN3 apply (+ skip connection)
        if self.nl is None:
            _bn_apply(self.bn3, self.h3, y, 0, "bn_apply", residual=xm if self.residual else None)
            return y
        _bn_apply(self.bn3, self.h3, self.nl_tail.l, 0, "bn_apply")   # l: the non-local input
        self.nl_tail.forward(xm, y, self.residual)
        return y

    def _expand_dw_train(self, xm):
        """Step 2 of TRAIN_EXPAND_DW_FUSED: h2 and BN2's batch statistics from x, W1 and BN1's
        batch coefficients (yamb_expand_dw_train_fwd); False, with nothing enqueued, when the
        kernel declines the shape (the caller then runs dw_fwd)."""
        global TRAIN_EXPAND_DW_CALLS
        conv = self.conv_dw[0]
        k, s = conv.kernel_size[0], conv.stride[0]
        a = nat.ExpandDwTrain()
        a.N, a.H, a.W, a.Cin, a.Chid = self.N, self.H, self.W, self.Cin, self.Chid
        a.kernel, a.stride, a.act, a.ldh = k, s, self.act, self.Chid
        a.x, a.w_expand = xm.data_ptr(), self.w_exp_bf.data_ptr()
        a.bn1_scale, a.bn1_shift = self.bn1.scale.data_ptr(), self.bn1.shift.data_ptr()
        a.w_dw, a.h2 = conv.weight.data_ptr(), self.h2.data_ptr()
        stats = self.bn2.fwd_struct(self.M_out)
        a.bn = C.pointer(stats)
        if not try_launch(nat.lib().yamb_expand_dw_train_fwd, a, "expand_dw_train",
                          2 * (self.M_in * self.Cin + self.M_out * self.Chid),
                          2 * self.Chid * (self.M_in * self.Cin + self.M_out * k * k)):
            return False
        TRAIN_EXPAND_DW_CALLS += 1
        return True

    def _dw_fwd_grouped(self):
        """Step 2 of TRAIN_MB_DW_GROUPED: every branch's depthwise in one
        yamb_depthwise_fwd_grouped launch, branch b with statistics slot b; False, with nothing
        enqueued, when the launcher declines (the caller then runs one dw_fwd per branch)."""
        global TRAIN_MB_DW_GROUPED_CALLS
        a = nat.DwFwdGrouped()
        a.nbranch = len(self.conv_dw)
        keep, nbytes, flops = [], 0, 0
        for b, ((c0, cb), conv) in enumerate(zip(self.bn2.slices, self.conv_dw)):
            s = slice(c0, c0 + cb)
            stats = self.bn2.fwd_struct(self.M_out, c0, cb, slot=b) if self.bn2.batch_stats \
                else None
            keep.append(stats)
            d, nb, fl = _dw_fwd_args(conv, (self.N, self.H, self.W), self.h1[:, s], self.h2[:, s],
                                     (self.bn1.scale[s], self.bn1.shift[s], self.act), stats)
            a.branch[b] = d
            nbytes, flops = nbytes + nb, flops + fl
        lib = nat.lib()
        rc = lib.yamb_depthwise_grouped_grids(C.byref(a), None)
        if rc == nat.EINVAL:
            return False
        nat.check(rc)
        if not try_launch(lib.yamb_depthwise_fwd_grouped, a, "dw_fwd_grouped", nbytes, flops):
            return False
        TRAIN_MB_DW_GROUPED_CALLS += 1
        return True

    def _dw_bwd_grouped(self, grads):
        """Step 4 of TRAIN_MB_DW_GROUPED: every branch's depthwise backward in one
        yamb_depthwise_bwd_grouped launch, branch b with statistics slot b; False, with nothing
        enqueued, when the launcher declines (the caller then runs one dw_bwd per branch)."""
        global TRAIN_MB_DW_GROUPED_CALLS
        a = nat.DwBwdGrouped()
        a.nbranch = len(self.conv_dw)
        keep, nbytes, flops = [], 0, 0
        for b, ((c0, cb), conv, dw) in enumerate(zip(self.bn2.slices, self.conv_dw, grads["dw"])):
            s = slice(c0, c0 + cb)
            stats = self.bn1.bwd_struct(self.M_in, grads["bn1"], c0, cb, slot=b)
            keep.append(stats)
            d, nb, fl = _dw_bwd_args(conv, (self.N, self.H, self.W), self.dz2[:, s], self.h2[:, s],
                                     (self.bn2.ca[s], self.bn2.cb[s], self.bn2.cc[s]), dw,
                                     self.h1[:, s], self.dz1[:, s],
                                     (self.bn1.scale[s], self.bn1.shift[s], self.act), None, stats)
            a.branch[b] = d
            nbytes, flops = nbytes + nb, flops + fl
        lib = nat.lib()
        rc = lib.yamb_depthwise_grouped_grids(None, C.byref(a))
        if rc == nat.EINVAL:
            return False
        nat.check(rc)
        if not try_launch(lib.yamb_depthwise_bwd_grouped, a, "dw_bwd_grouped", nbytes, flops):
            return False
        TRAIN_MB_DW_GROUPED_CALLS += 1
        return True

    def _se_backward(self, grads):
        """SE backward: dgate by a reduction kernel, the backward of the two fully connected layers
        (+ their parameter gradients) by yamb_se_fc_bwd, then
        dz2 = (d(a2*gate)*gate + dpool) * act'(z2) with the BN2-backward statistics."""
        lib = nat.lib()
        HW = self.Ho * self.Wo
        r = nat.SeBwdReduce()
        r.N, r.HW, r.C, r.ldd, r.ldh = self.N, HW, self.Chid, self.Chid, self.Chid
        r.dy, r.h = self.dz2.data_ptr(), self.h2.data_ptr()
        r.scale, r.shift, r.act = self.bn2.scale.data_ptr(), self.bn2.shift.data_ptr(), self.act
        r.dgate = self.dgate.data_ptr()
        launch(lib.yamb_se_bwd_reduce_bwd, r, "se_bwd_reduce", 4 * self.M_out * self.Chid)
        self._se_fc_backward(grads)
        for c0, cb in self.bn2.slices:
            s = slice(c0, c0 + cb)
            a = nat.SeBwdApply()
            a.M, a.C, a.ldd, a.ldh, a.ldz = self.M_out, cb, self.Chid, self.Chid, self.Chid
            a.rows_per_sample = HW
            a.dy = a.dz = self.dz2[:, s].data_ptr()
            a.h = self.h2[:, s].data_ptr()
            a.scale, a.shift = _at(self.bn2.scale, c0), _at(self.bn2.shift, c0)
            a.act = self.act
            a.gate, a.dpool = self.gate[:, s].data_ptr(), self.dpool[:, s].data_ptr()
            a.ldg = self.Chid
            a.bn = C.pointer(self.bn2.bwd_struct(self.M_out, grads["bn2"], c0, cb))
            launch(lib.yamb_se_bwd_apply_bwd, a, "se_bwd_apply", 6 * self.M_out * cb)

    def _se_backward_fused(self, grads):
        """SE backward of TRAIN_SE_FUSED: dgate and the per-(sample, channel) sums that the
        BatchNorm-2 backward statistics factor into by one reduction kernel, the FC backward, then
        the BatchNorm-2 finalize per slice from those sums, gate and dpool.  dz2 is not written:
        the depthwise backward forms it from dY (`_dw_bwd` with `se`)."""
        global TRAIN_SE_CALLS
        lib = nat.lib()
        HW = self.Ho * self.Wo
        sums = Workspace.get(self.dev).se_sums(4 * self.N * self.Chid)
        r = nat.SeBwdStats()
        r.N, r.HW, r.C, r.ldd, r.ldh = self.N, HW, self.Chid, self.Chid, self.Chid
        r.dy, r.h = self.dz2.data_ptr(), self.h2.data_ptr()
        r.scale, r.shift, r.act = self.bn2.scale.data_ptr(), self.bn2.shift.data_ptr(), self.act
        r.mean, r.invstd = self.bn2.mean.data_ptr(), self.bn2.invstd.data_ptr()
        r.dgate, r.sums = self.dgate.data_ptr(), sums.data_ptr()
        launch(lib.yamb_se_bwd_stats_bwd, r, "se_bwd_stats", 4 * self.M_out * self.Chid)
        self._se_fc_backward(grads)
        for c0, cb in self.bn2.slices:
            f = nat.SeBnBwdFinalize()
            f.N, f.C = self.N, cb
            f.sums, f.lds = sums.data_ptr() + 8 * c0, self.Chid
            f.gate, f.dpool, f.ldg = _at(self.gate, c0), _at(self.dpool, c0), self.Chid
            f.bn = C.pointer(self.bn2.bwd_struct(self.M_out, grads["bn2"], c0, cb))
            launch(lib.yamb_se_bn_bwd_finalize, f, "se_bn_bwd_finalize", 48 * self.N * cb)
        TRAIN_SE_CALLS += 1

    def _se_fc_backward(self, grads):
        """The backward of the two fully connected layers (+ their parameter gradients) from dgate:
        dpool for the BatchNorm-2 backward."""
        lib = nat.lib()
        se = self.se
        HW = self.Ho * self.Wo
        b = nat.SeFcBwd()
        b.N, b.C, b.R, b.act, b.inv_hw = self.N, self.Chid, self.se_r, self.se_act, 1.0 / HW
        b.dgate, b.gate = self.dgate.data_ptr(), self.gate.data_ptr()
        b.u, b.v, b.pooled = self.se_u.data_ptr(), self.se_v.data_ptr(), self.pooled.data_ptr()
        b.w_r, b.w_e = se.se_reduce.weight.data_ptr(), se.se_expand.weight.data_ptr()
        b.dpool, b.dt, b.du = self.dpool.data_ptr(), self.se_dt.data_ptr(), self.se_du.data_ptr()
        tg = grads["se"]
        b.g_wr, b.g_br, b.g_we, b.g_be = (tg[k].data_ptr() for k in ("wr", "br", "we", "be"))
        launch(lib.yamb_se_fc_bwd, b, "se_fc_bwd", 4 * self.N * self.Chid * 4,
               8 * self.N * self.Chid * self.se_r)

    # -- backward --------------------------------------------------------------------------------
    def backward(self, x, dy, grads, pre=None, pre_stats=None):
        """grads: dict with fp32 accumulation targets:
           'exp' [Chid,Cin], 'proj' [Cout,Chid], 'dw' list[[C,1,k,k]], 'bn1'/'bn2'/'bn3' lists of
           (dgamma, dbeta) per reference BN module.  Returns dx (channels_last bf16).  With the
           `pre` of the forward, dx is the gradient dz = da * act'(z) of the input BatchNorm's
           output, and `pre_stats` (a yamb_bn_bwd) takes that BatchNorm's backward statistics."""
        lib = nat.lib()
        bf = torch.bfloat16
        if self.dz2 is None:
            self.dh3 = torch.empty(self.M_out, self.Cout, device=self.dev, dtype=bf)
            self.dz2 = torch.empty(self.M_out, self.Chid, device=self.dev, dtype=bf)
            if self.expand:
                self.dz1 = torch.empty(self.M_in, self.Chid, device=self.dev, dtype=bf)
        xm = x.permute(0, 2, 3, 1).reshape(self.M_in, self.Cin)
        dym = dy.permute(0, 2, 3, 1).reshape(self.M_out, self.Cout)
        dym_skip = dym          # what the skip connection carries back to dx
        dx = torch.empty((self.N, self.Cin, self.H, self.W), device=self.dev, dtype=bf,
                         memory_format=torch.channels_last)
        if self.nl is not None:
            dym = self.nl_tail.backward(dym, grads)
        # 1. BN3 backward reduction -> ca3, cb3, cc3, dgamma3, dbeta3
        _bn_reduce(self.bn3.bwd_struct(self.M_out, grads["bn3"]), dym, self.h3, "bn_reduce")
        # 1b. dh3 = ca3*dy + cb3*h3 + cc3, formed once: both project GEMMs read it as a plain
        #     operand (as a loader transform it was re-read and re-formed for every n-block)
        _bn_bwd_apply(self.bn3, dym, self.h3, self.dh3, "bn3_bwd_apply")
        fork_ev = self._fork_event()
        # 2. project dgrad: da2 = dh3 * W3, dz2 = da2 * act'(z2), BN2-backward statistics, which
        #    the GEMM finalises for one BatchNorm module: one launch per branch slice.  With SE the
        #    GEMM writes d(a2*gate) over all channels; the gate / pooling gradients need a
        #    reduction over HW first, so act'/BN2-backward happen in se_bwd_apply afterwards
        se = self.se is not None
        for c0, cb in [(0, self.Chid)] if se else self.bn2.slices:
            s = slice(c0, c0 + cb)
            g = nat.Gemm()
            g.M, g.N, g.K = self.M_out, cb, self.Cout
            g.A, g.lda = self.dh3.data_ptr(), self.Cout
            g.B, g.ldb, g.b_mn_major = self.w_proj_bf[:, s].data_ptr(), self.Chid, 1
            g.D, g.ldd = self.dz2[:, s].data_ptr(), self.Chid
            if not se:
                g.epi = 1
                g.H, g.ldh = self.h2[:, s].data_ptr(), self.Chid
                g.h_scale, g.h_shift, g.h_act = _at(self.bn2.scale, c0), _at(self.bn2.shift, c0), \
                    self.act
                g.bn_bwd = C.pointer(self.bn2.bwd_struct(self.M_out, grads["bn2"], c0, cb))
            launch(lib.yamb_pointwise_gemm, g, "pw_project_dgrad",
                   2 * self.M_out * (self.Cout + (1 if se else 2) * cb),
                   2 * self.M_out * cb * self.Cout)
        se_fused = _se_fused(self.se)
        if se_fused:
            self._se_backward_fused(grads)
        elif se:
            self._se_backward(grads)
        # 3. project wgrad: dW3[Cout,Chid] += dh3^T * a2
        g = nat.Gemm()
        g.M, g.N, g.K = self.Cout, self.Chid, self.M_out
        g.a_mn_major = g.b_mn_major = 1
        g.A, g.lda = self.dh3.data_ptr(), self.Cout
        g.B, g.ldb = self.h2.data_ptr(), self.Chid
        g.b_xform, g.b_act = 1, self.act
        g.b_scale, g.b_shift = self.bn2.scale.data_ptr(), self.bn2.shift.data_ptr()
        if self.se is not None:
            g.b_gate, g.gate_rows_per_sample = self.gate.data_ptr(), self.Ho * self.Wo
        g.D, g.ldd = grads["proj"].data_ptr(), self.Chid
        g.epi = 2
        # needs only dh3 (step 1b) -> off the critical chain
        self._call_side(lib.yamb_pointwise_gemm, g, "pw_project_wgrad",
                        2 * self.M_out * (self.Cout + self.Chid),
                        2 * self.M_out * self.Chid * self.Cout, fork_ev, (self.dh3,))
        # 4. depthwise backward per branch, or of all branches in one launch (TRAIN_MB_DW_GROUPED)
        grouped = mb_dw_grouped(self) and not se_fused and self._dw_bwd_grouped(grads)
        for (c0, cb), conv, dw in [] if grouped else zip(self.bn2.slices, self.conv_dw,
                                                           grads["dw"]):
            s = slice(c0, c0 + cb)
            coef = (self.bn2.ca[s], self.bn2.cb[s], self.bn2.cc[s])
            se_args = (self.gate[:, s], self.dpool[:, s], self.bn2.scale[s], self.bn2.shift[s],
                       self.act) if se_fused else None
            if self.expand:
                _dw_bwd(conv, (self.N, self.H, self.W), self.dz2[:, s], self.h2[:, s], coef, dw,
                        self.h1[:, s], self.dz1[:, s], "dw_bwd",
                        pre=(self.bn1.scale[s], self.bn1.shift[s], self.act),
                        stats=self.bn1.bwd_struct(self.M_in, grads["bn1"], c0, cb), se=se_args)
            else:
                _dw_bwd(conv, (self.N, self.H, self.W), self.dz2[:, s], self.h2[:, s], coef, dw,
                        xm, dx, "dw_bwd", pre=pre, residual=dym_skip if self.residual else None,
                        stats=pre_stats, se=se_args)
        if not self.expand:
            return dx
        # 5+6. dh1 = ca1*dz1 + cb1*h1 + cc1 formed once, dx = dh1 * W1 (+ dy) and
        #      dW1 += dh1^T * x from the same staged tile: one read of dz1 and h1
        if self.expand_fused:
            a = nat.ExpandBwd()
            a.M, a.Cin, a.Chid = self.M_in, self.Cin, self.Chid
            a.dz1, a.h1 = self.dz1.data_ptr(), self.h1.data_ptr()
            a.ca, a.cb, a.cc = (t.data_ptr() for t in (self.bn1.ca, self.bn1.cb, self.bn1.cc))
            a.W1, a.x = self.w_exp_bf.data_ptr(), xm.data_ptr()
            a.residual = dym_skip.data_ptr() if self.residual else None
            a.dx, a.dW1 = dx.data_ptr(), grads["exp"].data_ptr()
            launch(lib.yamb_expand_bwd, a, "expand_bwd",
                   2 * self.M_in * (2 * self.Chid + self.Cin * (3 if self.residual else 2)),
                   4 * self.M_in * self.Chid * self.Cin)
            return dx
        fork2_ev = self._fork_event()   # dz1 and the BN1-backward coefficients exist from here on
        # 5. expand dgrad: dx = dh1 * W1 (+ dy)
        g = nat.Gemm()
        g.M, g.N, g.K = self.M_in, self.Cin, self.Chid
        g.A, g.lda = self.dz1.data_ptr(), self.Chid
        g.a_xform = 2
        g.a_scale, g.a_scale2, g.a_shift = self.bn1.ca.data_ptr(), self.bn1.cb.data_ptr(), \
            self.bn1.cc.data_ptr()
        g.A2, g.lda2 = self.h1.data_ptr(), self.Chid
        g.B, g.ldb, g.b_mn_major = self.w_exp_bf.data_ptr(), self.Cin, 1
        g.D, g.ldd = dx.data_ptr(), self.Cin
        if self.residual:
            g.residual, g.ldr = dym_skip.data_ptr(), self.Cout
        launch(lib.yamb_pointwise_gemm, g, "pw_expand_dgrad",
               2 * self.M_in * (2 * self.Chid + self.Cin * (2 if self.residual else 1)),
               2 * self.M_in * self.Chid * self.Cin)
        # 6. expand wgrad: dW1[Chid,Cin] += dh1^T * x
        g = nat.Gemm()
        g.M, g.N, g.K = self.Chid, self.Cin, self.M_in
        g.a_mn_major = g.b_mn_major = 1
        g.A, g.lda = self.dz1.data_ptr(), self.Chid
        g.a_xform = 2
        g.a_scale, g.a_scale2, g.a_shift = self.bn1.ca.data_ptr(), self.bn1.cb.data_ptr(), \
            self.bn1.cc.data_ptr()
        g.A2, g.lda2 = self.h1.data_ptr(), self.Chid
        g.B, g.ldb = xm.data_ptr(), self.Cin
        g.D, g.ldd = grads["exp"].data_ptr(), self.Cin
        g.epi = 2
        self._call_side(lib.yamb_pointwise_gemm, g, "pw_expand_wgrad",
                        2 * self.M_in * (2 * self.Chid + self.Cin),
                        2 * self.M_in * self.Chid * self.Cin, fork2_ev, (x,))
        return dx


# Expand-side backward: one yamb_expand_bwd launch where its plan covers the shape and the block
# has at least this many input pixels, else the dgrad GEMM + split-K wgrad GEMM.  Both paths give
# the same bits.  Measured on H100 (tests/gpu_expand_bwd_bench.py, BASELINE.md §5) the fused kernel
# is about twice as fast down to the smallest covered MobileNetV2 block, 25088 pixels (28 x 28 at
# N = 32: 98 slabs, fewer than the SMs); smaller maps are not measured and keep the two GEMMs.
EXPAND_BWD_MIN_M = 25088


def expand_bwd_fused(M_in, Cin, Chid):
    """True when BlockPlan.backward runs the expand-side backward as one yamb_expand_bwd launch."""
    if M_in < EXPAND_BWD_MIN_M or M_in >= 2 ** 31:
        return False
    a = nat.ExpandBwd()
    a.M, a.Cin, a.Chid = M_in, Cin, Chid
    info = nat.ExpandBwdPlanInfo()
    rc = nat.lib().yamb_expand_bwd_plan(C.byref(a), 1, C.byref(info))   # shape checks, no device
    if rc == nat.EINVAL:
        return False
    nat.check(rc)
    return True


def _bf16_operand(w, own, shape):
    """bf16 tensor-core operand of an fp32 master weight: the optimizer's mirror when it is
    provably fresh (same `_version` as when the mirror was last written), else a re-cast."""
    mirror = getattr(w, "_yamb_bf16", None)
    if mirror is None:
        own.copy_(w.view(shape))
        return own
    if getattr(w, "_yamb_bf16_version", None) != w._version:
        mirror.copy_(w)                       # stale: somebody wrote the master in place
        w._yamb_bf16_version = w._version
    return mirror.view(shape)


MAX_PLANS_PER_BLOCK = 2   # e.g. the training batch and the validation / calibration batch


def _plan_for(block, x):
    """BlockPlan (kernel sequence + intermediates) of `block` for this input shape.  At most
    MAX_PLANS_PER_BLOCK shapes are kept per block, least recently used first out: a partial last
    batch or another evaluation resolution no longer pins a whole extra activation set for ever
    (ADVICE r1)."""
    plans = block.__dict__.get("_yamb_plans")
    if plans is None:
        plans = block.__dict__["_yamb_plans"] = _ScratchDict()
    key = (tuple(x.shape), x.device.index)
    p = plans.pop(key, None)
    if p is None:
        p = BlockPlan(block, x)
        # dicts keep insertion order: oldest first.  A plan whose buffers a captured CUDA graph
        # addresses is never evicted (the graph holds raw pointers).
        for k in [k for k, q in plans.items() if not q.pinned][:max(0, len(plans) + 1 -
                                                                   MAX_PLANS_PER_BLOCK)]:
            plans.pop(k)
    if torch.cuda.is_current_stream_capturing():
        p.pinned = True
    plans[key] = p                              # (re-)insert as most recent
    return p


class _BlockFn(torch.autograd.Function):
    """autograd boundary of the fused block: forward/backward run the sm_90a kernel sequences.

    Parameter gradients go where `GradTargets` puts them: straight into the flat-arena optimizer's
    `.grad` views (autograd gets None), or into buffers of this backward returned to autograd."""

    @staticmethod
    def forward(ctx, x, block, *params):
        plan = _plan_for(block, x)
        y = plan.forward(x)
        ctx.block = block
        ctx.plan = plan
        ctx.generation = plan.generation
        ctx.save_for_backward(x)
        ctx.nparams = len(params)
        return y

    @staticmethod
    def backward(ctx, dy):
        plan, block = ctx.plan, ctx.block
        if plan.generation != ctx.generation:
            raise RuntimeError(
                "yamb: this block ran another forward before backward of the previous one; the "
                "saved intermediates were overwritten (one forward/backward in flight per block)")
        (x,) = ctx.saved_tensors
        dx, grads = run_backward(block, plan, x, dy)
        return (dx, None) + grads


def run_backward(block, plan, x, dy):
    """Backward kernel sequence of one block; returns dx and what autograd gets for
    `block.parameters()` (`GradTargets.result`)."""
    dy = to_nhwc_bf16(dy)
    gt = GradTargets(block.parameters())
    dx = plan.backward(x, dy, block_grads(gt, plan))
    if not DEFER_JOIN or gt.host_reads:
        join_side(plan.dev)
    return dx, gt.result()


def block_grads(gt, plan):
    """The `grads` argument of `plan.backward`: the accumulation targets in `gt` (a GradTargets
    over the block's parameters, possibly among others) of every parameter of the plan's block."""
    def bn_targets(bn):
        return [] if bn is None else [(gt.of(m.weight), gt.of(m.bias)) for m in bn.mods]

    g = {}
    if plan.expand:
        g["exp"] = gt.concat([c.weight for c in plan.conv_exp], 0, plan.concat_grads, "exp")
    g["proj"] = gt.concat([c.weight for c in plan.conv_proj], 1, plan.concat_grads, "proj")
    g["dw"] = [gt.of(c.weight) for c in plan.conv_dw]
    g["bn1"] = bn_targets(plan.bn1)
    g["bn2"] = bn_targets(plan.bn2)
    g["bn3"] = bn_targets(plan.bn3)
    if plan.se is not None:
        se = plan.se
        g["se"] = {"wr": gt.of(se.se_reduce.weight), "br": gt.of(se.se_reduce.bias),
                   "we": gt.of(se.se_expand.weight), "be": gt.of(se.se_expand.bias)}
    if plan.nl is not None:
        g["bn4"] = bn_targets(plan.bn4)
        g["nl_dw"] = gt.of(plan.nl.depthwise_conv.weight)
    return g


# ---- channel padding ---------------------------------------------------------------------------
# The kernels need every channel count to be a multiple of 8 (16-byte rows, TMA strides).  Searched
# networks (AtomNAS: hidden widths like [15, 23, 13], reference apps/searched/models/atomnas_c.yml)
# are run through a SHADOW block of the same class whose branch widths are rounded up to 8: the
# real parameters are scattered into the shadow's (padding: zero weights, gamma = beta = 0 so padded
# channels stay exactly 0 through BN + activation), the shadow runs the ordinary kernel sequence,
# gradients and running statistics are gathered back.  User-visible parameters are never padded.
def _ceil8(c):
    return (c + 7) // 8 * 8


def needs_padding(block):
    return any(c % 8 for c in block.channels)


class _PadShadow(Scratch):
    def __init__(self, block, device):
        from . import mobilenet_base as mb
        parts = block_parts(block)
        fused = parts.fused
        base = mb.InvertedResidualChannelsFused if fused else mb.InvertedResidualChannels
        self.real_ch = list(block.channels)
        self.pad_ch = [_ceil8(c) for c in self.real_ch]
        if block.input_dim % 8 or block.output_dim % 8:
            raise nat.NativeError("block input/output widths must be multiples of 8 (got %d -> %d)"
                                  % (block.input_dim, block.output_dim))
        if not block.expand:
            raise nat.NativeError("expand=False blocks need hidden == inp, a multiple of 8")
        kw = dict(active_fn=block.active_fn, batch_norm_kwargs=block.batch_norm_kwargs)
        if fused:
            kw.update(se_ratio=block.se_ratio, nl_c=block.nl_c, nl_s=block.nl_s)
        import logging
        lvl = logging.root.level
        self.shadow = base(block.input_dim, block.output_dim, block.stride, self.pad_ch,
                           list(block.kernel_sizes), block.expand, **kw).to(device)
        logging.root.setLevel(lvl)
        if parts.nl is not None:
            # the non-local norm (output width: never padded) is of the real block's class, which
            # the reference picks from FLAGS.nl_norm at construction time
            import copy
            self.shadow.nl_op.bn = copy.deepcopy(parts.nl.bn).to(device)
        for p in self.shadow.parameters():
            p.requires_grad_(False)
        real = dict(block.named_parameters())
        real.update(dict(block.named_buffers()))
        shad = dict(self.shadow.named_parameters())
        shad.update(dict(self.shadow.named_buffers()))
        tot_r, tot_p = sum(self.real_ch), sum(self.pad_ch)
        concat_idx, off = [], 0
        for c, cp in zip(self.real_ch, self.pad_ch):
            concat_idx.append(torch.arange(off, off + c))
            off += cp
        concat_idx = torch.cat(concat_idx)
        self.maps = {}
        for name, t in real.items():
            st = shad[name]
            if t.dim() == 0:
                self.maps[name] = None
                continue
            grids = []
            for d, (r, sdim) in enumerate(zip(t.shape, st.shape)):
                if r == sdim:
                    grids.append(torch.arange(r))
                elif r == tot_r and sdim == tot_p:
                    grids.append(concat_idx)          # concatenated hidden dimension
                elif r < sdim:
                    grids.append(torch.arange(r))     # one branch: its first r channels are real
                else:
                    raise nat.NativeError("cannot map %s %s -> %s" % (name, tuple(t.shape),
                                                                       tuple(st.shape)))
            pos = torch.arange(st.numel()).view(st.shape)
            for d, gi in enumerate(grids):
                pos = pos.index_select(d, gi)
            self.maps[name] = pos.reshape(-1).to(device)
        self.real_names = list(real.keys())
        self._build_flat(block, device)

    # ---- batched transfers ---------------------------------------------------------------------
    # Round 1 moved every parameter / buffer with its own index_copy_ (and every gradient with its
    # own index_select): ~100 tiny launches per padded block per step, 21 padded blocks in
    # AtomNAS-C+.  Now every floating-point shadow tensor is a view of ONE flat arena S and the
    # transfers are single gathers:
    #   push : S = cat(real tensors, [0, 1])[idx]          (pads -> 0, running_var pads -> 1)
    #   pull : real running statistics = S[stat_idx]       (one gather + one multi-tensor copy)
    #   grads: real gradients = cat(shadow gradients)[grad_idx]
    def _build_flat(self, block, device):
        real = dict(block.named_parameters())
        real.update(dict(block.named_buffers()))
        shad_p = dict(self.shadow.named_parameters())
        shad_b = dict(self.shadow.named_buffers())
        self.f_names = [n for n, t in real.items() if t.dim() > 0]          # float tensors
        self.i_names = [n for n, t in real.items() if t.dim() == 0]         # num_batches_tracked
        s_off, r_off, so, ro = {}, {}, 0, 0
        for n in self.f_names:
            st = shad_p[n] if n in shad_p else shad_b[n]
            s_off[n], r_off[n] = so, ro
            so += st.numel()
            ro += real[n].numel()
        self.S = torch.zeros(so, device=device, dtype=torch.float32)
        idx = torch.full((so,), ro, dtype=torch.long)               # default: the constant 0
        for n in self.f_names:
            st = shad_p[n] if n in shad_p else shad_b[n]
            if n.endswith("running_var"):
                idx[s_off[n]:s_off[n] + st.numel()] = ro + 1       # pads of a variance: 1
            m = self.maps[n].cpu()
            idx[s_off[n] + m] = r_off[n] + torch.arange(real[n].numel())
            view = self.S[s_off[n]:s_off[n] + st.numel()].view(st.shape)
            if n in shad_p:
                shad_p[n].data = view
            else:
                mod_name, _, key = n.rpartition(".")
                mod = self.shadow.get_submodule(mod_name) if mod_name else self.shadow
                mod._buffers[key] = view
        self.idx = idx.to(device)
        self.consts = torch.tensor([0.0, 1.0], device=device)
        # running statistics back to the real buffers
        self.stat_names = [n for n in self.f_names if n in shad_b]
        self.stat_idx = torch.cat([s_off[n] + self.maps[n].cpu() for n in self.stat_names]).to(device) \
            if self.stat_names else None
        self.stat_sizes = [real[n].numel() for n in self.stat_names]
        # gradients: positions of the real elements inside cat(shadow parameter gradients)
        self.p_names = [n for n in self.f_names if n in shad_p]
        g_off, go = {}, 0
        for n in self.p_names:
            g_off[n] = go
            go += shad_p[n].numel()
        self.grad_idx = torch.cat([g_off[n] + self.maps[n].cpu() for n in self.p_names]).to(device)
        self.grad_sizes = [real[n].numel() for n in self.p_names]

    def push(self, block):
        """real -> shadow (parameters, running statistics, BN / module modes): two launches."""
        real = dict(block.named_parameters())
        real.update(dict(block.named_buffers()))
        with torch.no_grad():
            src = torch.cat([real[n].detach().reshape(-1) for n in self.f_names] + [self.consts])
            torch.index_select(src, 0, self.idx, out=self.S)
            if self.i_names:
                shad_b = dict(self.shadow.named_buffers())
                for n in self.i_names:
                    shad_b[n].copy_(real[n])
        for (_, rm), (_, sm) in zip(block.named_modules(), self.shadow.named_modules()):
            sm.training = rm.training
            if isinstance(rm, (torch.nn.BatchNorm2d, torch.nn.InstanceNorm2d)):
                sm.momentum, sm.eps = rm.momentum, rm.eps

    def pull_stats(self, block):
        """shadow -> real running statistics after a training-mode forward."""
        if self.stat_idx is None:
            return
        real_b = dict(block.named_buffers())
        with torch.no_grad():
            flat = torch.index_select(self.S, 0, self.stat_idx)
            parts = flat.split(self.stat_sizes)
            torch._foreach_copy_([real_b[n].view(-1) for n in self.stat_names], list(parts))
            shad_b = dict(self.shadow.named_buffers())
            for n in self.i_names:
                real_b[n].copy_(shad_b[n])

    def gather_grads(self, gmap, block):
        """{id(shadow param): grad} -> list of real-shaped gradients in block.named_parameters()
        order (one cat + one gather)."""
        sp = dict(self.shadow.named_parameters())
        flat = torch.cat([gmap[id(sp[n])].reshape(-1).float() for n in self.p_names])
        real_flat = torch.index_select(flat, 0, self.grad_idx)
        parts = real_flat.split(self.grad_sizes)
        by_name = dict(zip(self.p_names, parts))
        return [by_name[n].view(p.shape) for n, p in block.named_parameters()]


class _PadFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, block, *params):
        sh = block.__dict__.get("_yamb_shadow")
        if sh is None:
            sh = _PadShadow(block, x.device)
            block.__dict__["_yamb_shadow"] = sh
        sh.push(block)
        plan = _plan_for(sh.shadow, x)
        y = plan.forward(x)
        sh.pull_stats(block)
        ctx.block, ctx.sh, ctx.plan, ctx.generation = block, sh, plan, plan.generation
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, dy):
        sh, plan, block = ctx.sh, ctx.plan, ctx.block
        if plan.generation != ctx.generation:
            raise RuntimeError("yamb: block re-entered before its backward (see _BlockFn)")
        (x,) = ctx.saved_tensors
        dx, shadow_grads = run_backward(sh.shadow, plan, x, dy)
        gmap = {id(p): g for p, g in zip(sh.shadow.parameters(), shadow_grads)}
        gt = GradTargets(block.parameters())
        gt.put_all(gt.params, sh.gather_grads(gmap, block))
        return (dx, None) + gt.result()


# ------------------------------------------------------------------------------------------------
# Stand-alone BatchNorm + activation of a ConvBNReLU (reference models/mobilenet_base.py:181-203)
# behind the stem 3x3 / head 1x1 convolution kernels or a convolution torch runs: raw conv output
# h [N,H,W,C] bf16 -> statistics kernel (+ finalize; skipped when the kernel that wrote h took the
# statistics) -> y = act(scale*h + shift); backward: statistics of dz = dy*act'(z) (+ finalize:
# dgamma, dbeta, ca/cb/cc) -> dh = ca*dz + cb*h + cc.
# ------------------------------------------------------------------------------------------------
class _BnActState(Scratch):
    def __init__(self, bn, dev):
        self.bn = _Bn([bn], dev)


def _bn_act_state(bn, dev):
    st = bn.__dict__.get("_yamb_bnact")
    if st is None or st.bn.dev != dev:
        st = _BnActState(bn, dev)
        bn.__dict__["_yamb_bnact"] = st
    return st


class _BnActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, h, bn, act, weight, bias, stats_taken):
        lib = nat.lib()
        st = _bn_act_state(bn, h.device)
        b = st.bn
        N, Cc, H, W = h.shape
        M = N * H * W
        hm = h.permute(0, 2, 3, 1).reshape(M, Cc)        # view of the channels_last storage
        if not b.batch_stats:
            with torch.no_grad():
                b.eval_coeffs()
        elif not stats_taken:
            s = nat.BnStats()
            s.M, s.C, s.ldh, s.h, s.bn = M, Cc, Cc, hm.data_ptr(), C.pointer(b.fwd_struct(M))
            launch(lib.yamb_bn_stats_fwd, s, "bn_stats", 2 * M * Cc)
        y = torch.empty_like(h, memory_format=torch.channels_last)
        _bn_apply(b, hm, y, act, "bn_apply")
        ctx.bn, ctx.act, ctx.st = bn, act, st
        # per-call copy of [scale, shift, mean, invstd]: another forward through this module before
        # the backward (eval / calibration pass, gradient accumulation) must not change what the
        # backward of THIS call sees (ADVICE r1)
        coef = torch.stack((b.scale, b.shift, b.mean, b.invstd)) if any(ctx.needs_input_grad) \
            else None
        ctx.save_for_backward(h, coef)
        return y

    @staticmethod
    def backward(ctx, dy):
        h, coef = ctx.saved_tensors
        bn, act, st = ctx.bn, ctx.act, ctx.st
        b = st.bn
        c_scale, c_shift, c_mean, c_invstd = (coef[i].data_ptr() for i in range(4))
        dy = to_nhwc_bf16(dy)
        N, Cc, H, W = h.shape
        M = N * H * W
        hm = h.permute(0, 2, 3, 1).reshape(M, Cc)
        dym = dy.permute(0, 2, 3, 1).reshape(M, Cc)
        gt = GradTargets((bn.weight, bn.bias))
        g = b.bwd_struct(M, [(gt.of(bn.weight), gt.of(bn.bias))])
        g.mean, g.invstd = c_mean, c_invstd      # this call's statistics, not the live buffers
        _bn_reduce(g, dym, hm, "bn_reduce", z=(c_scale, c_shift, act))
        dh = torch.empty_like(h, memory_format=torch.channels_last)
        _bn_bwd_apply(b, dym, hm, dh, "bn_bwd_apply", z=(c_scale, c_shift, act))
        return (dh, None, None) + gt.result() + (None,)


def bn_act_apply(bn, active_fn, h, stats_taken=False):
    """y = act(BatchNorm(h)) for a raw convolution output on CUDA (training or eval).
    stats_taken: the kernel that wrote h already took its batch statistics (a GEMM epilogue given
    `_bn_act_state(bn, dev).bn.fwd_struct`); ignored when `bn` folds its running statistics."""
    h = to_nhwc_bf16(h)
    if h.shape[1] % 8:
        raise nat.NativeError("bn_act: channel count must be a multiple of 8")
    return _BnActFn.apply(h, bn, act_code_of(active_fn), bn.weight, bn.bias, stats_taken)


# ---- eval mode: the whole block in one launch (csrc/block_eval.cu) ---------------------------------
# YAMB_EVAL_FUSED=0 keeps the four-launch sequence (folded coefficients) for every block.
EVAL_FUSED = os.environ.get("YAMB_EVAL_FUSED", "1") != "0"
EVAL_FUSED_CALLS = 0     # blocks that went through yamb_block_eval_fwd (tests / bench)

# ---- eval mode: the layers around the blocks (tail_ops.stem_eval / head_pool_eval) ----------------
# Off by default, so that a plain model.eval() forward launches what it always launched.  When True
# (trainer.EvalStep turns it on for its own forwards) the stem ConvBNReLU runs as one launch
# (yamb_stem_conv_eval_fwd) and the head ConvBNReLU + full-extent average pool as one launch
# (yamb_head_pool_eval_fwd), whenever no gradient is wanted, their BatchNorms use running statistics
# and the kernels cover the shape; otherwise the unfused sequence runs.
EVAL_TAIL_FUSED = False
EVAL_TAIL_CALLS = 0      # stem / head calls that went through the one-launch kernels (tests)

# ---- training mode: head BatchNorm + activation + average pool (tail_ops.head_pool_train) ---------
# Off by default: the pool's fixed summation order is not torch's, so turning it on changes the bits
# of a training step.  When True (trainer.TrainStep(fused_tail=True) turns it on for its own
# forwards and backwards) the head ConvBNReLU 1x1 followed by the full-extent average pool runs as
# the head GEMM + yamb_head_pool_train_fwd, backward yamb_head_pool_train_bwd, whenever the
# BatchNorm uses batch statistics and the kernels cover the shape: the activation and its broadcast
# gradient never reach HBM.  Otherwise the unfused sequence runs.
TRAIN_TAIL_FUSED = False
TRAIN_TAIL_CALLS = 0     # head calls that went through yamb_head_pool_train_fwd (tests)

# ---- training mode: stem BatchNorm + activation inside the first block (tail_ops.stem_block_train) --
# Off by default: the stem's statistics are summed in another order and, with Swish, dz is rounded
# after the act' product instead of before, so turning it on changes the bits of a training step.
# When True (trainer.TrainStep(fused_stem=True) turns it on for its own forwards and backwards) the
# stem ConvBNReLU and a first block without expansion or skip connection (the stem activation's
# only consumer, tail_ops.stem_block_fused_covered) run as one autograd function: the stem kernel
# takes the BatchNorm statistics of h, the block's depthwise applies BatchNorm + activation on load
# and writes dz with the BatchNorm-backward statistics, and the stem weight gradient forms dh on
# load; the activation, its gradient and dh never reach HBM.  Otherwise the unfused sequence runs.
TRAIN_STEM_FUSED = False
TRAIN_STEM_CALLS = 0     # stem + first block calls that went through stem_block_train (tests)

# ---- training mode: Squeeze-and-Excitation backward inside the depthwise backward ----------------
# Off by default: BatchNorm-2's backward statistics are summed from per-(sample, channel) factors
# instead of over the rounded dz2, so turning it on changes the bits of a training step (the same
# bits on every run).  When True (trainer.TrainStep(fused_se=True) turns it on for its own forwards
# and backwards) BlockPlan.backward of every block with SE runs se_bwd_stats -> se_fc_bwd ->
# se_bn_bwd_finalize -> depthwise_bwd_se instead of se_bwd_reduce -> se_fc_bwd -> se_bwd_apply ->
# depthwise_bwd: dz2 is formed by the depthwise backward while it stages dY and never reaches HBM.
TRAIN_SE_FUSED = False
TRAIN_SE_CALLS = 0       # block backwards that went through se_bwd_stats (tests)


# ---- training mode: expand + depthwise forward from x (yamb_expand_dw_train_fwd) ------------------
# Off by default.  When True (trainer.TrainStep(fused_expand_dw=True) turns it on for its own
# forwards) step 2 of BlockPlan.forward of a training block with one branch and an expansion whose
# shape EXPAND_DW_SHAPE_RULE accepts recomputes each depthwise input tile from x (TMA halo tile ->
# wgmma expand with the GEMM's bf16 W1 -> BatchNorm 1 + act -> stencil) instead of reading h1 back.
# The expand GEMM still writes h1 for the backward.  h2 has dw_fwd's bits; BatchNorm 2's statistics
# are summed in another order, so a step with it can differ from the default in the last bits.
# Multi-branch blocks, blocks without expansion and shapes the kernel declines run dw_fwd.
TRAIN_EXPAND_DW_FUSED = False
TRAIN_EXPAND_DW_CALLS = 0    # block forwards whose step 2 went through expand_dw_train (tests)
# EXPAND_DW_SHAPE_RULE sends a block down the path only when its kind (expand_dw_kind) is in
# EXPAND_DW_FASTER: the kinds that measured at least as fast as the expand GEMM's h1 read back by
# dw_fwd (tests/gpu_expand_dw_train_bench.py; BASELINE.md §5).  False: every covered block.
EXPAND_DW_SHAPE_RULE = True
EXPAND_DW_FASTER = frozenset()


def expand_dw_kind(block, H, W):
    """(k, stride, H, W, Cin, Chid) of a single-branch block with expansion on H x W inputs, the
    key of EXPAND_DW_SHAPE_RULE; None for a block the path never takes (several branches, no
    expansion)."""
    parts = block_parts(block)
    if not parts.expand_convs or len(parts.dws) != 1:
        return None
    conv = parts.dws[0][0]
    return (conv.kernel_size[0], conv.stride[0], H, W, parts.expand_convs[0].in_channels,
            conv.out_channels)


def _expand_dw_rule(kind):
    return kind is not None and (not EXPAND_DW_SHAPE_RULE or kind in EXPAND_DW_FASTER)


def expand_dw_selected(block, H, W):
    """Whether EXPAND_DW_SHAPE_RULE lets a training `block` on H x W inputs take the path."""
    return _expand_dw_rule(expand_dw_kind(block, H, W))


def expand_dw_fused(plan):
    """Whether step 2 of `plan` (a BlockPlan) tries yamb_expand_dw_train_fwd."""
    return (TRAIN_EXPAND_DW_FUSED and plan.expand and len(plan.conv_dw) == 1
            and plan.bn1.batch_stats and plan.bn2.batch_stats
            and _expand_dw_rule(plan.expand_dw_kind))


# ---- training mode: the depthwise of every branch in one launch each way ---------------------------
# Off by default.  When True (trainer.TrainStep(grouped_branches=True) turns it on for its own
# forwards and backwards) step 2 of BlockPlan.forward and step 4 of BlockPlan.backward of a
# training block with expansion and two or more branches launch yamb_depthwise_fwd_grouped /
# _bwd_grouped once instead of dw_fwd / dw_bwd once per branch.  Each CTA of the grouped grid runs
# what one CTA of a per-branch launch runs, so every output keeps its bits.  Only kinds
# MB_DW_SHAPE_RULE accepts take the path (none by default, see there).  Single-branch blocks,
# blocks without expansion, the backward with TRAIN_SE_FUSED (depthwise_bwd_se is not grouped) and
# arguments the launcher declines run the per-branch launches.
TRAIN_MB_DW_GROUPED = False
TRAIN_MB_DW_GROUPED_CALLS = 0    # grouped depthwise launches, forward and backward (tests)
# MB_DW_SHAPE_RULE groups a block only when its kind (mb_dw_kind) is in MB_DW_FASTER: the kinds
# whose grouped launches measured faster than the per-branch ones.  Empty: on an H100 most kinds
# of AtomNAS-C / C+ measured slower grouped and none faster in a way that survives run-to-run noise,
# and whole steps were 4-6 % slower (tests/gpu_mb_dw_grouped_bench.py; BASELINE.md §5).  False:
# every multi-branch block.
MB_DW_SHAPE_RULE = True
MB_DW_FASTER = frozenset()


def mb_dw_kind(block, H, W):
    """(kernel sizes, stride, H, W, Cin, hidden widths as run, padded to multiples of 8) of a
    block with an expansion and two or more branches, the key of MB_DW_SHAPE_RULE; None for a
    block that keeps its per-branch launches."""
    parts = block_parts(block)
    if not parts.expand_convs or len(parts.dws) < 2:
        return None
    return (tuple(conv.kernel_size[0] for conv, _ in parts.dws), parts.dws[0][0].stride[0], H, W,
            parts.expand_convs[0].in_channels, tuple(_ceil8(conv.out_channels)
                                                     for conv, _ in parts.dws))


def mb_dw_grouped(plan):
    """Whether step 2 / step 4 of `plan` (a BlockPlan) tries the grouped depthwise launch."""
    return (TRAIN_MB_DW_GROUPED and plan.expand and len(plan.conv_dw) >= 2
            and (not MB_DW_SHAPE_RULE or plan.mb_dw_kind in MB_DW_FASTER))


def mb_dw_group_plan(block, N, H, W):
    """The grouping of a training `block` on N x H x W inputs, as BlockPlan launches it: None when
    the block keeps its per-branch launches (one branch, no expansion), else a list with one dict
    per branch in launch order (the hidden tensor's channel order): its channel slice `c0`, `C`
    (BatchNorm-2 forward and BatchNorm-1 backward statistics of that slice, in statistics slot
    `slot`), `k` and `stride`."""
    parts = block_parts(block)
    if not parts.expand_convs or len(parts.dws) < 2:
        return None
    out, c0 = [], 0
    for b, (conv, _) in enumerate(parts.dws):
        cb = _ceil8(conv.out_channels)    # odd widths run as the padded shadow (_PadShadow)
        out.append({"slot": b, "c0": c0, "C": cb, "k": conv.kernel_size[0],
                    "stride": conv.stride[0]})
        c0 += cb
    return out


def _se_fused(se):
    """Whether BlockPlan.backward of a block whose SE module is `se` (None: none) runs the SE
    backward of TRAIN_SE_FUSED."""
    return TRAIN_SE_FUSED and se is not None


def se_backward_fused(block):
    """Whether the training backward of `block` runs the SE backward of TRAIN_SE_FUSED."""
    return _se_fused(block_parts(block).se)


def _eval_operands(block, dev, Chid, Cin, Cout, conv_e, conv_p):
    """bf16 tensor-core operands of the expand / project weights (the optimizer's mirrors when
    fresh, else block-owned copies kept in the `_yamb_eval` scratch that deepcopy / pickle drop)."""
    st = block.__dict__.get("_yamb_eval")
    if st is None:
        st = block.__dict__["_yamb_eval"] = _ScratchDict()
    key = dev.index
    own = st.get(key)
    if own is None:
        own = (torch.empty(Chid, Cin, device=dev, dtype=torch.bfloat16) if block.expand else None,
               torch.empty(Cout, Chid, device=dev, dtype=torch.bfloat16))
        st[key] = own
    with torch.no_grad():
        w1 = _bf16_operand(conv_e.weight, own[0], (Chid, Cin)) if block.expand else None
        w3 = _bf16_operand(conv_p.weight, own[1], (Cout, Chid))
    return w1, w3


def _block_eval_args(block, x, y, w1, w3, conv_d, bns, residual):
    """yamb_block_eval of one single-branch block; bns = (bn1 or None, bn2, bn3)."""
    N, Cin, H, W = x.shape
    a = nat.BlockEval()
    a.N, a.H, a.W = N, H, W
    a.Cin, a.Chid, a.Cout = Cin, block.channels[0], block.output_dim
    a.kernel, a.stride = block.kernel_sizes[0], block.stride
    a.act = act_code_of(block.active_fn)
    a.residual = 1 if residual else 0
    a.x, a.y = x.data_ptr(), nat.ptr(y)
    a.w_expand, a.w_project = nat.ptr(w1), w3.data_ptr()
    a.w_dw = conv_d.weight.data_ptr()
    for dst, bn in zip((a.bn1, a.bn2, a.bn3), bns):
        if bn is None:
            continue
        dst.gamma = nat.ptr(bn.weight)
        dst.beta = nat.ptr(bn.bias)
        dst.running_mean = bn.running_mean.data_ptr()
        dst.running_var = bn.running_var.data_ptr()
        dst.eps = bn.eps
    return a


def _block_eval_cost(block, x, Ho, Wo, residual, project=True):
    """(algorithmic bytes, flops) of one block_eval launch (engine.PROFILE bookkeeping)."""
    N, Cin, H, W = x.shape
    Chid, Cout, k = block.channels[0], block.output_dim, block.kernel_sizes[0]
    nbytes = 2 * N * H * W * Cin * (2 if residual else 1) + \
        (2 * N * Ho * Wo * Cout if project else 4 * N * Chid)
    flops = 2 * Chid * (N * H * W * (Cin if block.expand else 0) +
                        N * Ho * Wo * ((Cout if project else 0) + k ** 2))
    return nbytes, flops


# ---- one eval path for both block classes; InvertedResidualChannelsFused (AutoNL, AtomNAS) adds
# the SE gate and the non-local tail (reference models/mobilenet_base.py:330-342) -----------------
# Shape rule of the fused-class path, measured by tests/gpu_eval_bench_fused_class.py on one H100
# 80GB HBM3 (400 W power limit), N = 256, kernel time per block, new path vs the four-launch
# sequence.  5x5 blocks measured slower (AutoNL-L block 3, no SE: 1.08 vs 0.97 ms; block 14, SE:
# 0.50 vs 0.38 ms; block 21, SE + non-local: 1.06 vs 0.83 ms).  So did the blocks without the
# expansion at 112x112, whose four-launch sequence has no expand GEMM to save (AtomNAS-C+ block 1,
# SE: 1.64 vs 1.03 ms; AutoNL-L block 1: 0.85 vs 0.79 ms).  3x3 blocks with the expansion measured
# as fast or within 5 % (AutoNL-L block 8, non-local: 0.39 vs 0.50 ms; block 10, SE: 0.36 vs
# 0.42 ms; block 12, SE + non-local: 0.43 vs 0.42 ms).  k = 7 was not measured (no such block in
# AutoNL-L / AtomNAS-C+) and stays with k = 5.  False: every block the kernel covers takes the
# path (tests, tests/gpu_eval_bench_fused_class.py).
FUSED_CLASS_SHAPE_RULE = True

# ---- small batches: the hidden slices of every output tile split over a thread-block cluster -------
# (yamb_block_eval_cluster_fwd).  None: eval_cluster_size decides; 1, 2, 4 or 8: every block kernel
# launch of the eval path takes that cluster size (tests and tests/gpu_eval_latency_bench.py).
EVAL_CLUSTER = None
EVAL_CLUSTER_CALLS = 0   # block kernel launches that ran split over a cluster (tests)


def eval_tiles(k, stride, N, Ho, Wo, Cout):
    """Output tiles of one block_eval launch: the tile plan of csrc/block_eval.cuh
    (block_eval_launch_impl), which takes the geometry with the fewest tiles."""
    def tiles(toh, tow, ti):
        return -(-Ho // toh) * -(-Wo // tow) * -(-N // ti)
    if stride == 2:
        return tiles({3: 7, 5: 6, 7: 4}[k], 7, 1)
    if k == 7 or (Cout + 15) // 16 * 16 > 160:   # 7x7 depthwise, or a project wider than 160
        return tiles(7, 7, 1)
    return min(tiles(7, 16, 1), tiles(7, 7, 2))


def eval_cluster_size(k, stride, N, Ho, Wo, Chid, Cout, sms):
    """CTAs per cluster of one block_eval launch on a device with `sms` SMs: 1 (one CTA per tile)
    for a hidden dimension of fewer than 4 slices of 64 channels, else the largest S in {8, 4, 2}
    with tiles * S <= sms and at least S slices, else 1.  tests/gpu_eval_latency_bench.py on an
    H100 80GB HBM3 at 700 W (BASELINE.md, "Small-batch eval") measured the split slower than one
    CTA per tile on blocks of 2 or 3 slices (MobileNetV2 blocks 2-7 at N = 1: 37-43 vs 36-38 us)
    and faster on the wider ones (blocks 8-17: 42-46 vs 55-124 us)."""
    tiles, nc = eval_tiles(k, stride, N, Ho, Wo, Cout), -(-Chid // 64)
    if nc < 4:
        return 1
    for s in (8, 4, 2):
        if tiles * s <= sms and nc >= s:
            return s
    return 1


_SM_COUNT = {}


def _sm_count(dev):
    n = _SM_COUNT.get(dev.index)
    if n is None:
        n = _SM_COUNT[dev.index] = torch.cuda.get_device_properties(dev).multi_processor_count
    return n


def _bn_eval_ready(bn):
    return isinstance(bn, torch.nn.BatchNorm2d) and not bn.training and \
        bn.track_running_stats and bn.running_mean is not None


def _nl_norm_eval_ready(norm):
    """The non-local block's norm is a per-channel affine from running statistics."""
    if isinstance(norm, torch.nn.InstanceNorm2d):
        return _nl_norm_supported(norm) and not norm.training
    return _bn_eval_ready(norm)


def eval_supported(block, x):
    """True when the eval path covers this block for this call: no gradient wanted, every
    BatchNorm (the non-local block's included, or its tracked InstanceNorm) normalising with
    running statistics, one branch with a 3x3 / 5x5 / 7x7 depthwise (no expansion: 3x3 only),
    stride 1 or 2, widths that are multiples of 8 with Cin <= 256 and Cout <= 320.  Per class:
    InvertedResidualChannels (reference models/mobilenet_base.py:380-421) with k = 5 / 7 only for
    relu / relu6 / no activation (every block of MobileNetV2-1.0 and of Proxyless-mobile);
    InvertedResidualChannelsFused with any activation, with or without Squeeze-and-Excitation and
    a non-local block (every block of AutoNL-L, block 1 of AtomNAS-C+), minus the shapes
    FUSED_CLASS_SHAPE_RULE keeps on the four-launch sequence (8 AutoNL-L blocks take the path with
    it)."""
    if not EVAL_FUSED or torch.is_grad_enabled():
        return False
    if block.stride not in (1, 2) or len(block.channels) != 1:
        return False
    k = list(block.kernel_sizes)[0]
    cin, chid, cout = block.input_dim, block.channels[0], block.output_dim
    if k not in (3, 5, 7) or cin % 8 or chid % 8 or cout % 8 or cin > 256 or cout > 320:
        return False
    if not block.expand and (k != 3 or chid != cin):
        return False
    if x.dim() != 4 or x.shape[0] * x.shape[2] * x.shape[3] >= 2 ** 30:
        return False
    parts = block_parts(block)
    if not all(_bn_eval_ready(bn) for bn in parts.bn1s + [parts.dws[0][1], parts.bn3]):
        return False
    try:
        act = act_code_of(block.active_fn)
        if parts.se is not None:
            act_code_of(parts.se.active_fn)
    except ValueError:
        return False
    if not parts.fused:
        return k == 3 or act in (0, 1, 2)     # k = 5 / 7: built with relu / relu6 only
    if FUSED_CLASS_SHAPE_RULE and (k != 3 or not block.expand) and \
            not small_batch_listed(block, x.shape[0]):
        return False        # measured slower than the four-launch sequence at N = 256 (see above)
    nl = parts.nl
    if nl is not None:
        c = int(nl.nl_c * cout)
        if not _nl_norm_eval_ready(nl.bn) or c <= 0 or c % 2 or int(nl.nl_s) < 1:
            return False
    return True


def _block_eval_launch(fn, fn_cluster, a, cluster, tag, nbytes, flops):
    """One block kernel launch, split over clusters of `cluster` CTAs when cluster > 1 and the
    tile plan with the exchanged partials fits shared memory, else unsplit.  True when split."""
    global EVAL_CLUSTER_CALLS
    if cluster > 1 and try_launch(lambda st, s: fn_cluster(st, cluster, s), a, tag + "_cluster",
                                  nbytes, flops):
        EVAL_CLUSTER_CALLS += 1
        return True
    launch(fn, a, tag, nbytes, flops)
    return False


def eval_forward(block, x):
    """y = block(x) in eval mode; x channels_last bf16 on CUDA.  C-ABI calls: the block kernel
    (1); with SE the pool pass and the gate FCs first (3); with a non-local block the kernel writes
    l = BN3(h3) and the non-local tail follows (+4)."""
    global EVAL_FUSED_CALLS
    dev = x.device
    N, Cin, H, W = x.shape
    parts = block_parts(block)
    conv_e, bn1 = (parts.expand_convs[0], parts.bn1s[0]) if block.expand else (None, None)
    (conv_d, bn2), conv_p, bn3 = parts.dws[0], parts.project_convs[0], parts.bn3
    se, nl = parts.se, parts.nl
    Chid, Cout, stride = block.channels[0], block.output_dim, block.stride
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    w1, w3 = _eval_operands(block, dev, Chid, Cin, Cout, conv_e, conv_p)
    bf = torch.bfloat16
    y = torch.empty((N, Cout, Ho, Wo), device=dev, dtype=bf, memory_format=torch.channels_last)
    # the block kernel's output: y itself, or l = BN3(h3) (no skip connection) for the non-local tail
    residual = block.use_res_connect and nl is None
    tail = None
    if nl is not None:
        st = block.__dict__["_yamb_eval"]
        bn4 = st.get(("bn4", dev.index))
        if bn4 is None:
            bn4 = st[("bn4", dev.index)] = _Bn([nl.bn], dev)
        tail = _NlTail(nl, bn4, N, Ho, Wo, Cout, dev)
    out = y if tail is None else tail.l
    a = _block_eval_args(block, x, out, w1, w3, conv_d, (bn1, bn2, bn3), residual)
    cluster = EVAL_CLUSTER if EVAL_CLUSTER is not None else eval_cluster_size(
        block.kernel_sizes[0], stride, N, Ho, Wo, Chid, Cout, _sm_count(dev))
    lib = nat.lib()
    if se is not None:
        # gate = sigmoid(W_e act(W_r mean_HW(a2) + b_r) + b_e): pool pass, then the two FCs
        R = se.se_reduce.weight.shape[0]
        pooled = torch.empty(N, Chid, device=dev, dtype=torch.float32)
        gate = torch.empty(N, Chid, device=dev, dtype=torch.float32)
        uv = torch.empty(2, N, R, device=dev, dtype=torch.float32)
        a.pooled = pooled.data_ptr()
        _block_eval_launch(lib.yamb_block_eval_pool_fwd, lib.yamb_block_eval_cluster_pool_fwd, a,
                           cluster, "block_eval_pool",
                           *_block_eval_cost(block, x, Ho, Wo, False, project=False))
        _se_fc(se, pooled, uv[0], uv[1], gate)
        a.pooled = None
        a.gate = gate.data_ptr()
    _block_eval_launch(lib.yamb_block_eval_fwd, lib.yamb_block_eval_cluster_fwd, a, cluster,
                       "block_eval", *_block_eval_cost(block, x, Ho, Wo, residual))
    if tail is not None:
        xm = x.permute(0, 2, 3, 1).reshape(N * H * W, Cin)    # view, NHWC matrix
        tail.forward(xm, y.permute(0, 2, 3, 1).reshape(N * Ho * Wo, Cout), block.use_res_connect)
    EVAL_FUSED_CALLS += 1
    return y


# ---- eval mode: multi-branch blocks (several depthwise kernel sizes: AtomNAS) in one launch ---------
# (csrc/block_eval_mb.cu).  Off by default, so that a plain model.eval() forward launches what it
# always launched: the hidden channels are regrouped by kernel size, so the project sums in another
# order and the block's output differs from the four-launch sequence in the last bits.  When True
# (trainer.EvalStep(fused_multi_branch=True) turns it on for its evaluation forwards) every block
# eval_mb_supported covers runs as yamb_block_eval_mb_pack + the block kernel (+ the SE pool pass
# and gate FCs first).
EVAL_MULTI_BRANCH = False
EVAL_MB_CALLS = 0        # blocks that went through yamb_block_eval_mb_fwd (tests / bench)

# Kinds of block (K_MAX, stride, fused class; the path has the expansion only) that measured at
# least as fast as the four-launch sequence with its _PadShadow gathers.
# tests/gpu_eval_bench_multi_branch.py on one H100 80GB HBM3 (700 W power limit), N = 256, device time
# of every multi-branch block of AtomNAS-C / C+ summed per kind, new path vs four launches:
# (7, 1, unfused) 5.24 vs 4.71 ms over 16 blocks (faster on the 14x14 / 7x7 blocks of < 400 hidden
# channels, slower on the 56x56 / 28x28 ones and the widest), (7, 2, unfused) 3.57 vs 2.86 ms,
# (5, 1, unfused) 0.41 vs 0.40 ms; with SE the pool pass runs the expand and the stencil a second
# time: (7, 1, fused) 13.97 vs 6.90 ms, (7, 2, fused) 10.37 vs 3.90, (5, 1, fused) 1.16 vs 0.50.
# No kind measured at least as fast, so none takes the path by default.  MB_SHAPE_RULE = False:
# every block the kernel covers takes it (tests, the benchmark).
MB_SHAPE_RULE = True
MB_FASTER = frozenset()

# ---- small batches (trainer.EvalStep(small_batch=True) sets EVAL_SMALL_BATCH around its evaluation
# forwards).  Both shape rules above were measured at N = 256, where the work is bandwidth-bound;
# at N = 1 a block is one or a few tiles and the count of serial launches decides.  While the
# switch is on:
#   - eval_forward_mb splits the packed hidden slices of every tile over a thread-block cluster
#     (yamb_block_eval_mb_cluster_fwd, the size from eval_cluster_size as in eval_forward);
#   - a multi-branch block whose kind is listed in SMALL_BATCH_FASTER takes the multi-branch path
#     at N <= the listed bound, whatever EVAL_MULTI_BRANCH / MB_SHAPE_RULE say;
#   - a fused-class block FUSED_CLASS_SHAPE_RULE keeps on the four-launch sequence takes the
#     one-launch path at N <= the bound of its kind.
# Kinds (small_batch_kind): ("mb", K_MAX, stride, fused class) and ("fused", k, stride, expansion).
# SMALL_BATCH_RULE = False: every kind at every N (tests, tests/gpu_eval_latency_bench_searched.py).
# SMALL_BATCH_FASTER: tests/gpu_eval_latency_bench_searched.py --rule off on one H100 80GB HBM3
# (700 W power limit), every block of the kind alone in a CUDA graph, summed per kind, at
# N = 1, 2, 4, 8, 16, 64; a kind is listed up to the largest measured N at which it and every smaller
# N were faster than the default in every config that has it (BASELINE.md §5, "Small-batch eval of
# the searched networks").  At N = 1: AtomNAS-C (7, 1) 1.64 -> 0.64 ms over 16 blocks, AtomNAS-C+
# (7, 1, SE) 2.06 -> 1.54 ms, AutoNL-L 5x5 stride 1 0.83 -> 0.63 ms.  The SE kinds lose from
# N = 16 / 64 on, where their pool pass's recompute costs more than the launches it saves.
EVAL_SMALL_BATCH = False
EVAL_MB_CLUSTER_CALLS = 0   # multi-branch block kernel launches split over a cluster (tests)
SMALL_BATCH_RULE = True
SMALL_BATCH_FASTER = (      # ((kind, max N), ...)
    (("mb", 5, 1, False), 64), (("mb", 7, 1, False), 64), (("mb", 7, 2, False), 64),
    (("mb", 5, 1, True), 16), (("mb", 7, 1, True), 16), (("mb", 7, 2, True), 8),
    (("fused", 3, 1, False), 4), (("fused", 5, 1, True), 64), (("fused", 5, 2, True), 64),
)


def small_batch_kind(block):
    """What SMALL_BATCH_FASTER decides on: ("mb",) + mb_kind for a multi-branch block, else
    ("fused", k, stride, expansion)."""
    if len(block.channels) > 1:
        return ("mb",) + mb_kind(block)
    return ("fused", list(block.kernel_sizes)[0], block.stride, bool(block.expand))


def small_batch_listed(block, N):
    """True while EVAL_SMALL_BATCH is on for a block whose kind SMALL_BATCH_FASTER lists with a
    bound >= N (any block when SMALL_BATCH_RULE is off)."""
    if not EVAL_SMALL_BATCH:
        return False
    if not SMALL_BATCH_RULE:
        return True
    kind = small_batch_kind(block)
    return any(k == kind and N <= n for k, n in SMALL_BATCH_FASTER)


MbLayout = collections.namedtuple("MbLayout", "map Chid kmax groups")


def mb_layout(kernel_sizes, channels):
    """Packed hidden dimension of a multi-branch block: the branches in order of decreasing kernel
    size (stable), each padded to a multiple of 8 channels.  map[j] = (branch << 16) | channel, or
    -1 for a padded channel; groups = [(k, first packed channel)] of decreasing k."""
    ks, cs = list(kernel_sizes), list(channels)
    m, groups = [], []
    for i in sorted(range(len(ks)), key=lambda i: -ks[i]):
        if not groups or groups[-1][0] != ks[i]:
            groups.append((ks[i], len(m)))
        m += [(i << 16) | c for c in range(cs[i])] + [-1] * (_ceil8(cs[i]) - cs[i])
    return MbLayout(m, len(m), groups[0][0], groups)


def mb_kind(block):
    """(K_MAX, stride, fused class) of a multi-branch block: what MB_SHAPE_RULE decides on."""
    return max(block.kernel_sizes), block.stride, hasattr(block, "expand_conv")


def eval_mb_supported(block, x):
    """True when the multi-branch eval path covers this block for this call: EVAL_MULTI_BRANCH on,
    no gradient wanted, 2 or 3 branches with the expansion and 3x3 / 5x5 / 7x7 depthwise kernels
    (K_MAX 5 or 7), stride 1 or 2, Cin <= 256 and Cout <= 320 multiples of 8, every BatchNorm
    normalising with running statistics and one eps, an activation the kernel has, no non-local
    block, and a kind MB_SHAPE_RULE lets through, or one small_batch_listed lets through while
    EVAL_SMALL_BATCH is on."""
    if not ((EVAL_MULTI_BRANCH or EVAL_SMALL_BATCH) and EVAL_FUSED) or torch.is_grad_enabled():
        return False
    ks, chans = list(block.kernel_sizes), list(block.channels)
    if not 2 <= len(ks) <= 3 or not block.expand or block.stride not in (1, 2):
        return False
    if any(k not in (3, 5, 7) for k in ks) or max(ks) == 3 or min(chans) <= 0:
        return False
    cin, cout = block.input_dim, block.output_dim
    if cin % 8 or cout % 8 or cin > 256 or cout > 320:
        return False
    if x.dim() != 4 or x.shape[0] * x.shape[2] * x.shape[3] >= 2 ** 30:
        return False
    parts = block_parts(block)
    bns = parts.bn1s + [bn for _, bn in parts.dws] + [parts.bn3]
    if not all(_bn_eval_ready(bn) for bn in bns) or len({bn.eps for bn in bns[:-1]}) != 1:
        return False
    if parts.nl is not None:
        return False
    try:
        act_code_of(block.active_fn)
        if parts.se is not None:
            act_code_of(parts.se.active_fn)
    except ValueError:
        return False
    if small_batch_listed(block, x.shape[0]):
        return True
    return EVAL_MULTI_BRANCH and (not MB_SHAPE_RULE or mb_kind(block) in MB_FASTER)


def _mb_state(block, dev, R):
    """The packed tensors of a multi-branch block on `dev` and its layout (device index map
    included), in the `_yamb_eval` scratch that deepcopy / pickle drop."""
    st = block.__dict__.get("_yamb_eval")
    if st is None:
        st = block.__dict__["_yamb_eval"] = _ScratchDict()
    key = ("mb", dev.index)
    ms = st.get(key)
    if ms is None:
        lay = mb_layout(block.kernel_sizes, block.channels)
        Chid, K, Cin, Cout = lay.Chid, lay.kmax, block.input_dim, block.output_dim
        f32, bf = torch.float32, torch.bfloat16
        ms = st[key] = {
            "layout": lay,
            "map": torch.tensor(lay.map, dtype=torch.int32, device=dev),
            "w1": torch.empty(Chid, Cin, device=dev, dtype=bf),
            "w3": torch.empty(Cout, Chid, device=dev, dtype=bf),
            "wdw": torch.empty(Chid, K, K, device=dev, dtype=f32),
            "bn1": torch.empty(4, Chid, device=dev, dtype=f32),
            "bn2": torch.empty(4, Chid, device=dev, dtype=f32),
            "se": (torch.empty(R, Chid, device=dev, dtype=f32),
                   torch.empty(Chid, R, device=dev, dtype=f32),
                   torch.empty(Chid, device=dev, dtype=f32)) if R else None,
        }
    return ms


def _mb_pack_args(block, parts, ms):
    """yamb_block_eval_mb_pack_args of a multi-branch block into its packed tensors `ms`."""
    lay, se = ms["layout"], parts.se
    pk = nat.BlockEvalMbPack()
    pk.Cin, pk.Cout = block.input_dim, block.output_dim
    pk.R = se.se_reduce.weight.shape[0] if se is not None else 0
    pk.nbranch = len(block.channels)
    c0 = 0
    for i, (k, c) in enumerate(zip(block.kernel_sizes, block.channels)):
        b = pk.branch[i]
        b.k, b.C = k, c
        b.ld = sum(block.channels) if parts.fused else c
        conv_d, bn2 = parts.dws[i]
        if parts.fused:     # one expand conv / BN1 / project conv: the branch's rows / columns
            w1, bn1, w3 = parts.expand_convs[0].weight, parts.bn1s[0], parts.project_convs[0].weight
            off = c0
        else:
            w1, bn1, w3 = parts.expand_convs[i].weight, parts.bn1s[i], parts.project_convs[i].weight
            off = 0
        b.w_expand = w1.data_ptr() + 4 * off * pk.Cin
        for dst, bn, o in ((b.bn1, bn1, off), (b.bn2, bn2, 0)):
            dst.gamma, dst.beta = _at(bn.weight, o), _at(bn.bias, o)
            dst.running_mean, dst.running_var = _at(bn.running_mean, o), _at(bn.running_var, o)
            dst.eps = bn.eps
        b.w_dw = conv_d.weight.data_ptr()
        b.w_project = w3.data_ptr() + 4 * off
        if se is not None:
            b.se_reduce = se.se_reduce.weight.data_ptr() + 4 * off
            b.se_expand = se.se_expand.weight.data_ptr() + 4 * off * pk.R
            b.se_expand_bias = se.se_expand.bias.data_ptr() + 4 * off
        c0 += c
    pk.Chid, pk.kmax = lay.Chid, lay.kmax
    pk.map = ms["map"].data_ptr()
    pk.w_expand, pk.w_project, pk.w_dw = ms["w1"].data_ptr(), ms["w3"].data_ptr(), ms["wdw"].data_ptr()
    pk.bn1, pk.bn2 = ms["bn1"].data_ptr(), ms["bn2"].data_ptr()
    if se is not None:
        pk.se_reduce, pk.se_expand, pk.se_expand_bias = (t.data_ptr() for t in ms["se"])
    return pk


def eval_forward_mb(block, x):
    """y = block(x) in eval mode for a multi-branch block; x channels_last bf16 on CUDA.  C-ABI
    calls: the packing kernel and the block kernel (2); with SE the pool pass and the gate FCs
    between them (+2).  While EVAL_SMALL_BATCH is on, the block kernel and the pool pass split
    over a cluster as eval_forward's do."""
    global EVAL_MB_CALLS, EVAL_MB_CLUSTER_CALLS
    dev = x.device
    N, Cin, H, W = x.shape
    parts = block_parts(block)
    se = parts.se
    R = se.se_reduce.weight.shape[0] if se is not None else 0
    ms = _mb_state(block, dev, R)
    lay = ms["layout"]
    Chid, Cout, stride = lay.Chid, block.output_dim, block.stride
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    lib = nat.lib()
    pk = _mb_pack_args(block, parts, ms)
    w_bytes = 4 * Chid * (Cin + Cout + lay.kmax ** 2 + 8 + 2 * R)
    launch(lib.yamb_block_eval_mb_pack, pk, "block_eval_mb_pack", 2 * w_bytes, 0)
    y = torch.empty((N, Cout, Ho, Wo), device=dev, dtype=torch.bfloat16,
                    memory_format=torch.channels_last)
    m = nat.BlockEvalMb()
    a = m.base
    a.N, a.H, a.W = N, H, W
    a.Cin, a.Chid, a.Cout = Cin, Chid, Cout
    a.kernel, a.stride = lay.kmax, stride
    a.act = act_code_of(block.active_fn)
    a.residual = 1 if block.use_res_connect else 0
    a.x, a.y = x.data_ptr(), y.data_ptr()
    a.w_expand, a.w_project, a.w_dw = ms["w1"].data_ptr(), ms["w3"].data_ptr(), ms["wdw"].data_ptr()
    eps = parts.dws[0][1].eps
    for dst, t in ((a.bn1, ms["bn1"]), (a.bn2, ms["bn2"])):
        dst.gamma, dst.beta, dst.running_mean, dst.running_var = (r.data_ptr() for r in t)
        dst.eps = eps
    bn3 = parts.bn3
    a.bn3.gamma, a.bn3.beta = nat.ptr(bn3.weight), nat.ptr(bn3.bias)
    a.bn3.running_mean, a.bn3.running_var = bn3.running_mean.data_ptr(), bn3.running_var.data_ptr()
    a.bn3.eps = bn3.eps
    m.ngroups = len(lay.groups)
    for i, (k, c0) in enumerate(lay.groups):
        m.group_k[i], m.group_c0[i] = k, c0
    flops = 2 * Chid * N * (H * W * Cin + Ho * Wo * Cout) + \
        2 * N * Ho * Wo * sum(k * k * c for k, c in zip(block.kernel_sizes, block.channels))
    act_bytes = 2 * N * H * W * Cin * (2 if a.residual else 1)
    cluster = 1
    if EVAL_SMALL_BATCH:
        cluster = EVAL_CLUSTER if EVAL_CLUSTER is not None else eval_cluster_size(
            lay.kmax, stride, N, Ho, Wo, Chid, Cout, _sm_count(dev))
    if se is not None:
        pooled = torch.empty(N, Chid, device=dev, dtype=torch.float32)
        gate = torch.empty(N, Chid, device=dev, dtype=torch.float32)
        uv = torch.empty(2, N, R, device=dev, dtype=torch.float32)
        a.pooled = pooled.data_ptr()
        if _block_eval_launch(lib.yamb_block_eval_mb_pool_fwd, lib.yamb_block_eval_mb_cluster_pool_fwd,
                              m, cluster, "block_eval_mb_pool", act_bytes + 4 * N * Chid, flops):
            EVAL_MB_CLUSTER_CALLS += 1
        _se_fc(se, pooled, uv[0], uv[1], gate, packed=ms["se"])
        a.pooled = None
        a.gate = gate.data_ptr()
    if _block_eval_launch(lib.yamb_block_eval_mb_fwd, lib.yamb_block_eval_mb_cluster_fwd, m, cluster,
                          "block_eval_mb", act_bytes + 2 * N * Ho * Wo * Cout, flops):
        EVAL_MB_CLUSTER_CALLS += 1
    EVAL_MB_CALLS += 1
    return y


def block_apply(block, x):
    """Forward of a reference-compatible block module through the sm_90a path."""
    if not x.is_cuda:
        raise nat.NativeError(
            "the inverted-residual block runs only on CUDA sm_90a (no CPU fallback); got a %s "
            "tensor" % x.device)
    x = to_nhwc_bf16(x)
    if eval_supported(block, x):
        return eval_forward(block, x)
    if eval_mb_supported(block, x):
        return eval_forward_mb(block, x)
    params = list(block.parameters())
    if needs_padding(block):
        return _PadFn.apply(x, block, *params)
    return _BlockFn.apply(x, block, *params)
