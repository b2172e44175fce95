"""Host-side sequencing of the sm_90a kernels for one inverted-residual block.

A `BlockPlan` owns the HBM-resident intermediates of one block for one input shape
(NHWC bf16 [pixels, channels] matrices) and the pre-built C-ABI argument structs; `block_apply`
is the autograd entry the modules in `mobilenet_base.py` call.  Kernel order (train mode):

  forward   expand GEMM (+BN1 stats) -> depthwise (BN1+act on load, +BN2 stats)
            -> project GEMM (BN2+act operand transform, +BN3 stats) -> BN3 apply (+x)
  backward  BN3 reduce -> project dgrad GEMM (BN3-bwd operand transform, act'/BN2-bwd epilogue)
            + project wgrad GEMM -> depthwise bwd (BN2-bwd on load, fused wgrad, act'/BN1-bwd
            epilogue) -> expand dgrad GEMM (+dy) + expand wgrad GEMM

Reference semantics: models/mobilenet_base.py:446-451 (unfused), :330-342 (fused) and their
torch.autograd backward.  No tensor between the 1x1 convs is ever normalised in HBM: BatchNorm +
activation are applied by the consumer on load.
"""
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


def lib_fn(name):
    return getattr(nat.lib(), name)


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
    """Scratch of the statistics-producing kernels: the global fp32 accumulator of the per-channel
    sums (2*C floats, zero between launches — the last CTA of every launch returns it to zero) and
    the arrival counter.  The kernels of ONE stream serialise on it, so there is one per
    (device, stream): blocks driven from two streams at the same time (VERDICT r1) do not share."""
    _per_stream = {}

    def __init__(self, device):
        lib = nat.lib()
        self.max_ctas = lib.yamb_max_ctas()
        if self.max_ctas <= 0:
            raise nat.NativeError("no CUDA device visible to libyamb200 (there is no CPU path)")
        self.max_c = 4096
        self.partials = torch.zeros(4 * self.max_c, device=device, dtype=torch.float32)
        self.counter = torch.zeros(4, device=device, dtype=torch.int32)

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


def _nl_norm_supported(norm):
    """The non-local block's norms the sm_90a path runs (reference get_nl_norm_fn,
    models/mobilenet_base.py:472-481): BatchNorm2d (`nl_norm: nn.BatchNorm`, the default) and the
    tracked affine InstanceNorm2d (`nl_norm: nn.InstanceNorm`)."""
    if isinstance(norm, torch.nn.BatchNorm2d):
        return True
    return isinstance(norm, torch.nn.InstanceNorm2d) and norm.affine and \
        norm.track_running_stats and norm.running_mean is not None


class _NlTail:
    """Non-local block (reference models/mobilenet_base.py:158-173) behind a BatchNorm output l,
    for one shape: y = norm(dw3x3(f)) + l (+ x), f = (W/H) theta (phi^T g).  Owns l, f, h (bf16
    [N*H*W, C]) and F (fp32 [N][c][C]); `forward` is the four launches of the training plan and of
    the eval path alike.

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
        self.keep = []

    def gram(self, X, I, Y, sub, alpha, G, tag):
        g = nat.NlGram()
        g.N, g.H, g.W, g.sub = self.N, self.H, self.W, sub
        g.X, g.ldx, g.I = X.data_ptr(), self.C, I
        g.Y, g.ldy, g.J = Y.data_ptr(), self.C, self.C
        g.alpha, g.G = alpha, G.data_ptr()
        self.keep.append(g)
        launch(lib_fn("yamb_nl_gram_fwd"), g, tag, 4 * self.M * self.C // (sub * sub))

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
        self.keep.append(r)
        launch(lib_fn("yamb_nl_rowmat_fwd"), r, tag, 4 * self.M * self.C // (sub * sub))

    def forward(self, xm, y, residual, bn_fwd_struct=None):
        """self.l -> y.  bn_fwd_struct(bn, count): the yamb_bn_fwd of BN4 when it normalises with
        batch statistics (train mode); otherwise BN4 is folded from its running statistics."""
        lib = nat.lib()
        self.keep = []
        Cc, c = self.C, self.cr
        instance = self.instance and self.bn4.batch_stats
        if instance and self.H * self.W == 1:
            raise nat.NativeError("non-local block: InstanceNorm in training mode needs more than "
                                  "one pixel per channel (the map is 1x1)")
        self.used_instance_stats = instance
        # F = phi^T g over the sub-sampled pixels; f = (W/H) theta F
        self.gram(self.l, c, self.l, self.sub, 1.0, self.F, "nl_gram")
        self.rowmat(self.l, c, self.F, Cc, 1, Cc, 1, self.scale, self.f, "nl_apply")
        # depthwise 3x3 (no activation before it) + BN4 statistics
        d = nat.DwFwd()
        d.N, d.H, d.W, d.C, d.ldc, d.k, d.stride = self.N, self.H, self.W, Cc, Cc, 3, 1
        d.x = self.f.data_ptr()
        d.w = self.nl.depthwise_conv.weight.data_ptr()
        d.y = self.h.data_ptr()
        if instance:
            pass                               # statistics per sample: yamb_instance_norm_fwd
        elif self.bn4.batch_stats:
            d.bn = C.pointer(bn_fwd_struct(self.bn4, self.M))
        else:
            self.bn4.eval_coeffs()
        launch(lib.yamb_depthwise_fwd, d, "nl_dw_fwd", 4 * Cc * self.M, 2 * self.M * Cc * 9)
        if instance:
            self._instance_forward(xm, y, residual)
            return
        # y = BN4(h) + l (+ x)
        a = nat.BnApply()
        a.M, a.C = self.M, Cc
        a.ldh = a.ldr = a.ldy = Cc
        a.h, a.scale, a.shift = self.h.data_ptr(), self.bn4.scale.data_ptr(), \
            self.bn4.shift.data_ptr()
        a.act = 0
        a.residual = self.l.data_ptr()
        if residual:
            a.residual2, a.ldr2 = xm.data_ptr(), Cc
        a.y = y.data_ptr()
        self.keep += [d, a]
        launch(lib.yamb_bn_apply_fwd, a, "nl_bn_apply", 2 * self.M * Cc * (4 if residual else 3))

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
        self.keep.append(s)
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
        self.keep.append(s)
        launch(nat.lib().yamb_instance_norm_bwd, s, "nl_in_bwd", 2 * self.M * Cc * 5)


class BlockPlan:
    def __init__(self, block, x):
        dev = x.device
        self.dev = dev
        self.ws = Workspace.get(dev)
        self.lib = nat.lib()
        N, Cin, H, W = x.shape
        self.N, self.H, self.W, self.Cin = N, H, W, Cin
        self.stride = block.stride
        # pad=(k-1)//2, odd k: out = floor((H-1)/s)+1
        self.Ho = (H - 1) // self.stride + 1
        self.Wo = (W - 1) // self.stride + 1
        self.Cout = block.output_dim
        self.channels = list(block.channels)
        self.ks = list(block.kernel_sizes)
        self.expand = bool(block.expand)
        self.residual = bool(block.use_res_connect)
        self.act = act_code_of(block.active_fn)
        self.fused = hasattr(block, "expand_conv")
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
        self.dz2 = None
        self.dz1 = None
        # ---- modules ----
        if self.fused:
            self.conv_exp = [block.expand_conv[0]] if self.expand else []
            bn1 = [block.expand_conv[1]] if self.expand else []
            dws = [list(op.children())[-1] for op in block.depth_ops]
            self.conv_proj = [block.project_conv[0]]
            bn3 = block.project_conv[1]
            self.se = block.se_op if type(block.se_op).__name__ != "Identity" else None
            self.nl = block.nl_op if type(block.nl_op).__name__ != "Identity" else None
        else:
            if self.expand:
                self.conv_exp = [op[0][0] for op in block.ops]
                bn1 = [op[0][1] for op in block.ops]
                dws = [op[1] for op in block.ops]
                self.conv_proj = [op[2] for op in block.ops]
            else:
                self.conv_exp, bn1 = [], []
                dws = [op[0] for op in block.ops]
                self.conv_proj = [op[1] for op in block.ops]
            bn3 = block.pw_bn
        if not self.fused:
            self.se = None
            self.nl = None
        if self.nl is not None:
            # non-local block (reference models/mobilenet_base.py:131-178) between BN3 and the skip
            nl = self.nl
            if not _nl_norm_supported(nl.bn):
                raise nat.NativeError(
                    "non-local block: the sm_90a path runs nn.BatchNorm2d and "
                    "nn.InstanceNorm2d(affine=True, track_running_stats=True) as nl_norm (got %r)"
                    % nl.bn)
            self.nl_tail = tail = _NlTail(nl, _Bn([nl.bn], dev), N, self.Ho, self.Wo, Cout, dev)
            self.nl_cr, self.nl_sub, self.nl_scale = tail.cr, tail.sub, tail.scale
            self.nl_l, self.nl_f, self.nl_h, self.nl_F = tail.l, tail.f, tail.h, tail.F
            self.nl_dF = None
            self.nl_df = None
            self.nl_dl = None
            self.nl_in_dh = None
            self.bn4 = tail.bn4
            self.g_nl = torch.zeros_like(nl.depthwise_conv.weight, dtype=torch.float32)
        if self.se is not None:
            self.se_act = act_code_of(self.se.active_fn)
            self.se_r = self.se.se_reduce.weight.shape[0]
            self.se_u = _f32(N * self.se_r, dev).view(N, self.se_r)
            self.se_v = _f32(N * self.se_r, dev).view(N, self.se_r)
            self.se_du = _f32(N * self.se_r, dev).view(N, self.se_r)
            self.se_dt = _f32(N * Chid, dev).view(N, Chid)
            self.g_se = {k: torch.zeros_like(t, dtype=torch.float32) for k, t in (
                ("wr", self.se.se_reduce.weight), ("br", self.se.se_reduce.bias),
                ("we", self.se.se_expand.weight), ("be", self.se.se_expand.bias))}
            self.pooled = _f32(N * Chid, dev).view(N, Chid)
            self.gate = _f32(N * Chid, dev).view(N, Chid)
            self.dgate = _f32(N * Chid, dev).view(N, Chid)
            self.dpool = _f32(N * Chid, dev).view(N, Chid)
        self.conv_dw = [d[0] for d in dws]
        self.bn1 = _Bn(bn1, dev) if self.expand else None
        self.bn2 = _Bn([d[1] for d in dws], dev)
        self.bn3 = _Bn([bn3], dev)
        # ---- bf16 tensor-core operands + fp32 gradient accumulators ----
        self.w_exp_bf = torch.empty(Chid, Cin, device=dev, dtype=bf) if self.expand else None
        self.w_proj_bf = torch.empty(Cout, Chid, device=dev, dtype=bf)
        self.w_exp_own, self.w_proj_own = self.w_exp_bf, self.w_proj_bf
        self.g_exp = _f32(Chid * Cin, dev).view(Chid, Cin) if self.expand else None
        self.g_proj = _f32(Cout * Chid, dev).view(Cout, Chid)
        self.g_dw = [torch.zeros_like(c.weight, dtype=torch.float32) for c in self.conv_dw]
        self.generation = 0
        self.pinned = False
        self._keep = []

    # -- helpers -------------------------------------------------------------------------------
    def _bn_fwd_struct(self, bn, count, c0=0, C=None):
        """yamb_bn_fwd for channels [c0, c0+C) of stage `bn` (per-branch slice for depthwise)."""
        C = bn.C if C is None else C
        s = nat.BnFwd()
        ws = Workspace.get(self.dev)     # of the stream this launch goes to
        s.partials = ws.partials.data_ptr()
        s.counter = ws.counter.data_ptr()
        if bn.single:
            m = bn.mods[0]
            g, b = m.weight, m.bias
            rm, rv, nbt = m.running_mean, m.running_var, m.num_batches_tracked
            off = c0
        else:
            # slice == exactly one reference BN module
            idx = [i for i, (s0, n) in enumerate(bn.slices) if s0 == c0 and n == C]
            if len(idx) != 1:
                raise nat.NativeError("BatchNorm slice does not match a reference module")
            m = bn.mods[idx[0]]
            g, b = m.weight, m.bias
            rm, rv, nbt = m.running_mean, m.running_var, m.num_batches_tracked
            off = 0
        f4 = 4
        s.gamma = g.data_ptr() + off * f4 if g is not None else None
        s.beta = b.data_ptr() + off * f4 if b is not None else None
        s.eps = bn.eps
        s.momentum = bn.momentum_value()
        if m.track_running_stats and rm is not None:
            s.running_mean = rm.data_ptr() + off * f4
            s.running_var = rv.data_ptr() + off * f4
            s.num_batches_tracked = nbt.data_ptr() if nbt is not None else None
        s.scale = bn.scale.data_ptr() + c0 * f4
        s.shift = bn.shift.data_ptr() + c0 * f4
        s.mean = bn.mean.data_ptr() + c0 * f4
        s.invstd = bn.invstd.data_ptr() + c0 * f4
        s.count = count
        self._keep.append(s)
        return s

    def _bn_bwd_struct(self, bn, count, grads, c0=0, C=None):
        C = bn.C if C is None else C
        s = nat.BnBwd()
        ws = Workspace.get(self.dev)     # of the stream this launch goes to
        s.partials = ws.partials.data_ptr()
        s.counter = ws.counter.data_ptr()
        f4 = 4
        if bn.single:
            mi, off = 0, c0
        else:
            mi = [i for i, (s0, n) in enumerate(bn.slices) if s0 == c0 and n == C][0]
            off = 0
        m = bn.mods[mi]
        s.gamma = m.weight.data_ptr() + off * f4 if m.weight is not None else None
        s.mean = bn.mean.data_ptr() + c0 * f4
        s.invstd = bn.invstd.data_ptr() + c0 * f4
        dg, db = grads[mi]
        s.dgamma = dg.data_ptr() + off * f4 if dg is not None else None
        s.dbeta = db.data_ptr() + off * f4 if db is not None else None
        s.ca = bn.ca.data_ptr() + c0 * f4
        s.cb = bn.cb.data_ptr() + c0 * f4
        s.cc = bn.cc.data_ptr() + c0 * f4
        s.count = count
        s.use_batch_stats = 1 if bn.batch_stats else 0
        self._keep.append(s)
        return s

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

    def _call(self, fn, st, tag="", nbytes=0, flops=0):
        launch(fn, st, tag, nbytes, flops)

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
    def forward(self, x):
        """x: channels_last bf16 [N,Cin,H,W]; returns channels_last bf16 [N,Cout,Ho,Wo]."""
        lib = self.lib
        self._keep = []
        self.generation += 1
        self._refresh_weights()
        xm = x.permute(0, 2, 3, 1).reshape(self.M_in, self.Cin)  # view, NHWC matrix
        y = torch.empty((self.N, self.Cout, self.Ho, self.Wo), device=self.dev,
                        dtype=torch.bfloat16, memory_format=torch.channels_last)
        # 1. expand 1x1 + BN1 statistics
        if self.expand:
            g = nat.Gemm()
            g.M, g.N, g.K = self.M_in, self.Chid, self.Cin
            g.A, g.lda = xm.data_ptr(), self.Cin
            g.B, g.ldb = self.w_exp_bf.data_ptr(), self.Cin
            g.D, g.ldd = self.h1.data_ptr(), self.Chid
            if self.bn1.batch_stats:
                if self.bn1.single:
                    g.bn_fwd = C.pointer(self._bn_fwd_struct(self.bn1, self.M_in))
                    self._call(lib.yamb_pointwise_gemm, g, "pw_expand_fwd",
                               2 * self.M_in * (self.Cin + self.Chid),
                               2 * self.M_in * self.Cin * self.Chid)
                else:
                    # per-branch BN modules: one finalize per branch slice is done by the GEMM only
                    # for a single module; otherwise run the statistics per slice via N-slices
                    self._gemm_sliced_stats(g, self.bn1, self.M_in)
            else:
                self.bn1.eval_coeffs()
                self._call(lib.yamb_pointwise_gemm, g, "pw_expand_fwd",
                           2 * self.M_in * (self.Cin + self.Chid),
                           2 * self.M_in * self.Cin * self.Chid)
        # 2. depthwise per branch (BN1+act applied on load) + BN2 statistics
        if not self.bn2.batch_stats:
            self.bn2.eval_coeffs()
        c0 = 0
        for b, (cb, k) in enumerate(zip(self.channels, self.ks)):
            d = nat.DwFwd()
            # hidden pitch; when not expanding hidden == inp, so x has the same pitch
            d.N, d.H, d.W, d.C, d.ldc, d.k, d.stride = self.N, self.H, self.W, cb, self.Chid, k, \
                self.stride
            if self.expand:
                d.x = self.h1.data_ptr() + c0 * 2
                d.in_scale = self.bn1.scale.data_ptr() + c0 * 4
                d.in_shift = self.bn1.shift.data_ptr() + c0 * 4
                d.in_act = self.act
            else:
                d.x = xm.data_ptr()
            d.w = self.conv_dw[b].weight.data_ptr()
            d.y = self.h2.data_ptr() + c0 * 2
            if self.bn2.batch_stats:
                d.bn = C.pointer(self._bn_fwd_struct(self.bn2, self.M_out, c0, cb))
            self._call(lib.yamb_depthwise_fwd, d, "dw_fwd", 2 * cb * (self.M_in + self.M_out),
                       2 * self.M_out * cb * k * k)
            c0 += cb
        # 2b. Squeeze-and-Excitation gate (reference mobilenet_base.py:110-113): spatial mean of
        #     a2 = act(bn2(h2)) by a kernel, the two fully connected layers + sigmoid by another,
        #     the gate applied inside the project GEMM's operand transform
        if self.se is not None:
            sp = nat.SePool()
            sp.N, sp.HW, sp.C, sp.ldh = self.N, self.Ho * self.Wo, self.Chid, self.Chid
            sp.h, sp.scale, sp.shift, sp.act = self.h2.data_ptr(), self.bn2.scale.data_ptr(), \
                self.bn2.shift.data_ptr(), self.act
            sp.pooled = self.pooled.data_ptr()
            self._call(lib.yamb_se_pool_fwd, sp, "se_pool", 2 * self.M_out * self.Chid)
            se = self.se
            # the two fully connected layers on the pooled [N, C] vectors (fp32, like the reference
            # keeps them) + sigmoid: one launch (csrc/se_fc.cu)
            f = nat.SeFc()
            f.N, f.C, f.R, f.act = self.N, self.Chid, self.se_r, self.se_act
            f.pooled = self.pooled.data_ptr()
            f.w_r, f.b_r = se.se_reduce.weight.data_ptr(), se.se_reduce.bias.data_ptr()
            f.w_e, f.b_e = se.se_expand.weight.data_ptr(), se.se_expand.bias.data_ptr()
            f.u, f.v, f.gate = self.se_u.data_ptr(), self.se_v.data_ptr(), self.gate.data_ptr()
            self._keep.append(f)
            self._call(lib.yamb_se_fc_fwd, f, "se_fc", 4 * self.N * self.Chid * 2,
                       4 * self.N * self.Chid * self.se_r)
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
            g.bn_fwd = C.pointer(self._bn_fwd_struct(self.bn3, self.M_out))
        else:
            self.bn3.eval_coeffs()
        self._call(lib.yamb_pointwise_gemm, g, "pw_project_fwd",
                   2 * self.M_out * (self.Chid + self.Cout),
                   2 * self.M_out * self.Chid * self.Cout)
        # 4. BN3 apply (+ skip connection)
        a = nat.BnApply()
        a.M, a.C = self.M_out, self.Cout
        a.ldh = a.ldr = a.ldy = self.Cout
        a.h, a.scale, a.shift = self.h3.data_ptr(), self.bn3.scale.data_ptr(), \
            self.bn3.shift.data_ptr()
        a.act = 0
        if self.nl is None:
            a.residual = xm.data_ptr() if self.residual else None
            a.y = y.data_ptr()
            self._call(lib.yamb_bn_apply_fwd, a, "bn_apply",
                       2 * self.M_out * self.Cout * (3 if self.residual else 2))
            return y
        a.y = self.nl_l.data_ptr()              # l = BN3(h3): the non-local block's input
        self._call(lib.yamb_bn_apply_fwd, a, "bn_apply", 4 * self.M_out * self.Cout)
        self.nl_tail.forward(xm, y, self.residual, self._bn_fwd_struct)
        return y

    # -- non-local block (reference models/mobilenet_base.py:158-173) ------------------------------
    def _nl_gram(self, X, I, Y, sub, alpha, G, tag):
        self.nl_tail.gram(X, I, Y, sub, alpha, G, tag)

    def _nl_rowmat(self, X, K, Mat, sk, so, O, sub, alpha, out, tag, base=None, accumulate=0):
        self.nl_tail.rowmat(X, K, Mat, sk, so, O, sub, alpha, out, tag, base, accumulate)

    def _nl_backward(self, dym, grads):
        """dy -> dl (gradient of the BN3 output): BN4 backward, depthwise 3x3 backward, the two
        products' backward, plus the `+ l` pass-through."""
        lib = self.lib
        Cc, c, bf = self.Cout, self.nl_cr, torch.bfloat16
        if self.nl_df is None:
            self.nl_df = torch.empty(self.M_out, Cc, device=self.dev, dtype=bf)
            self.nl_dl = torch.empty(self.M_out, Cc, device=self.dev, dtype=bf)
            self.nl_dF = _f32(self.N * c * Cc, self.dev)
        tail = self.nl_tail
        d = nat.DwBwd()
        d.N, d.H, d.W, d.C, d.ldc, d.k, d.stride = self.N, self.Ho, self.Wo, Cc, Cc, 3, 1
        if tail.used_instance_stats:
            # InstanceNorm with per-sample statistics: its backward writes dh (bf16), which the
            # depthwise backward takes with the identity coefficients ca = 1, cb = cc = 0
            if self.nl_in_dh is None:
                self.nl_in_dh = torch.empty(self.M_out, Cc, device=self.dev, dtype=bf)
                self.nl_ones = torch.ones(Cc, device=self.dev, dtype=torch.float32)
                self.nl_zeros = _f32(Cc, self.dev)
            tail.instance_backward(dym, self.nl_in_dh, grads["bn4"])
            d.dz, d.h = self.nl_in_dh.data_ptr(), self.nl_h.data_ptr()
            d.ca, d.cb, d.cc = self.nl_ones.data_ptr(), self.nl_zeros.data_ptr(), \
                self.nl_zeros.data_ptr()
        else:
            r = nat.BnReduce()
            r.M, r.C, r.lddy, r.ldh = self.M_out, Cc, Cc, Cc
            r.dy, r.h = dym.data_ptr(), self.nl_h.data_ptr()
            r.bn = C.pointer(self._bn_bwd_struct(self.bn4, self.M_out, grads["bn4"]))
            self._call(lib.yamb_bn_reduce_bwd, r, "nl_bn_reduce", 4 * self.M_out * Cc)
            d.dz, d.h = dym.data_ptr(), self.nl_h.data_ptr()
            d.ca, d.cb, d.cc = self.bn4.ca.data_ptr(), self.bn4.cb.data_ptr(), \
                self.bn4.cc.data_ptr()
        d.w = self.nl.depthwise_conv.weight.data_ptr()
        d.dw = grads["nl_dw"].data_ptr()
        d.x = self.nl_f.data_ptr()
        d.dx = self.nl_df.data_ptr()
        self._keep.append(d)
        self._call(lib.yamb_depthwise_bwd, d, "nl_dw_bwd", 8 * Cc * self.M_out,
                   4 * self.M_out * Cc * 9)
        # dF = (W/H) theta^T df (all pixels);  dl = dy + [dtheta | 0];  sub-sampled rows += dphi, dg
        self._nl_gram(self.nl_l, c, self.nl_df, 1, self.nl_scale, self.nl_dF, "nl_gram_bwd")
        self._nl_rowmat(self.nl_df, Cc, self.nl_F, 1, Cc, c, 1, self.nl_scale, self.nl_dl,
                        "nl_dtheta", base=dym)
        self._nl_rowmat(self.nl_l, Cc, self.nl_dF, 1, Cc, c, self.nl_sub, 1.0, self.nl_dl,
                        "nl_dphi", accumulate=1)
        self._nl_rowmat(self.nl_l, c, self.nl_dF, Cc, 1, Cc, self.nl_sub, 1.0, self.nl_dl,
                        "nl_dg", accumulate=1)
        return self.nl_dl

    def _gemm_sliced_stats(self, g, bn, count):
        """Expand GEMM whose output channels belong to several BN modules: one GEMM per module
        slice (N-slices of the weight), each finalising its own BatchNorm."""
        lib = self.lib
        for (c0, cb) in bn.slices:
            gs = nat.Gemm()
            C.memmove(C.byref(gs), C.byref(g), C.sizeof(nat.Gemm))
            gs.N = cb
            gs.B = g.B + c0 * g.ldb * 2
            gs.D = g.D + c0 * 2
            gs.bn_fwd = C.pointer(self._bn_fwd_struct(bn, count, c0, cb))
            self._call(lib.yamb_pointwise_gemm, gs, "pw_expand_fwd", 2 * gs.M * (gs.K + cb),
                       2 * gs.M * gs.K * cb)

    def _se_backward(self, grads):
        """SE backward: dgate by a reduction kernel, the backward of the two fully connected layers
        (+ their parameter gradients) by yamb_se_fc_bwd, then
        dz2 = (d(a2*gate)*gate + dpool) * act'(z2) with the BN2-backward statistics."""
        lib = self.lib
        se = self.se
        HW = self.Ho * self.Wo
        r = nat.SeBwdReduce()
        r.N, r.HW, r.C, r.ldd, r.ldh = self.N, HW, self.Chid, self.Chid, self.Chid
        r.dy, r.h = self.dz2.data_ptr(), self.h2.data_ptr()
        r.scale, r.shift, r.act = self.bn2.scale.data_ptr(), self.bn2.shift.data_ptr(), self.act
        r.dgate = self.dgate.data_ptr()
        self._call(lib.yamb_se_bwd_reduce_bwd, r, "se_bwd_reduce", 4 * self.M_out * self.Chid)
        b = nat.SeFcBwd()
        b.N, b.C, b.R, b.act, b.inv_hw = self.N, self.Chid, self.se_r, self.se_act, 1.0 / HW
        b.dgate, b.gate = self.dgate.data_ptr(), self.gate.data_ptr()
        b.u, b.v, b.pooled = self.se_u.data_ptr(), self.se_v.data_ptr(), self.pooled.data_ptr()
        b.w_r, b.w_e = se.se_reduce.weight.data_ptr(), se.se_expand.weight.data_ptr()
        b.dpool, b.dt, b.du = self.dpool.data_ptr(), self.se_dt.data_ptr(), self.se_du.data_ptr()
        tg = grads["se"]
        b.g_wr, b.g_br, b.g_we, b.g_be = (tg[k].data_ptr() for k in ("wr", "br", "we", "be"))
        self._keep.append(b)
        self._call(lib.yamb_se_fc_bwd, b, "se_fc_bwd", 4 * self.N * self.Chid * 4,
                   8 * self.N * self.Chid * self.se_r)
        for (c0, cb) in self.bn2.slices:
            a = nat.SeBwdApply()
            a.M, a.C, a.ldd, a.ldh, a.ldz = self.M_out, cb, self.Chid, self.Chid, self.Chid
            a.rows_per_sample = HW
            a.dy = self.dz2.data_ptr() + c0 * 2
            a.h = self.h2.data_ptr() + c0 * 2
            a.scale = self.bn2.scale.data_ptr() + c0 * 4
            a.shift = self.bn2.shift.data_ptr() + c0 * 4
            a.act = self.act
            a.gate = self.gate.data_ptr() + c0 * 4
            a.dpool = self.dpool.data_ptr() + c0 * 4
            a.ldg = self.Chid
            a.dz = self.dz2.data_ptr() + c0 * 2
            a.bn = C.pointer(self._bn_bwd_struct(self.bn2, self.M_out, grads["bn2"], c0, cb))
            self._call(lib.yamb_se_bwd_apply_bwd, a, "se_bwd_apply", 6 * self.M_out * cb)

    # -- backward --------------------------------------------------------------------------------
    def backward(self, x, dy, grads):
        """grads: dict with fp32 accumulation targets:
           'exp' [Chid,Cin], 'proj' [Cout,Chid], 'dw' list[[C,1,k,k]], 'bn1'/'bn2'/'bn3' lists of
           (dgamma, dbeta) per reference BN module.  Returns dx (channels_last bf16)."""
        lib = self.lib
        self._keep = []
        bf = torch.bfloat16
        if self.dz2 is None:
            self.dz2 = torch.empty(self.M_out, self.Chid, device=self.dev, dtype=bf)
            if self.expand:
                self.dz1 = torch.empty(self.M_in, self.Chid, device=self.dev, dtype=bf)
        xm = x.permute(0, 2, 3, 1).reshape(self.M_in, self.Cin)
        dym = dy.permute(0, 2, 3, 1).reshape(self.M_out, self.Cout)
        dym_skip = dym          # what the skip connection carries back to dx
        dx = torch.empty((self.N, self.Cin, self.H, self.W), device=self.dev, dtype=bf,
                         memory_format=torch.channels_last)
        if self.nl is not None:
            dym = self._nl_backward(dym, grads)
        # 1. BN3 backward reduction -> ca3, cb3, cc3, dgamma3, dbeta3
        r = nat.BnReduce()
        r.M, r.C, r.lddy, r.ldh = self.M_out, self.Cout, self.Cout, self.Cout
        r.dy, r.h = dym.data_ptr(), self.h3.data_ptr()
        r.bn = C.pointer(self._bn_bwd_struct(self.bn3, self.M_out, grads["bn3"]))
        self._call(lib.yamb_bn_reduce_bwd, r, "bn_reduce", 4 * self.M_out * self.Cout)
        fork_ev = self._fork_event()
        # 2. project dgrad: da2 = dh3 * W3, dz2 = da2 * act'(z2), BN2-backward statistics
        g = nat.Gemm()
        g.M, g.N, g.K = self.M_out, self.Chid, self.Cout
        g.A, g.lda = dym.data_ptr(), self.Cout
        g.a_xform = 2
        g.a_scale, g.a_scale2, g.a_shift = self.bn3.ca.data_ptr(), self.bn3.cb.data_ptr(), \
            self.bn3.cc.data_ptr()
        g.A2, g.lda2 = self.h3.data_ptr(), self.Cout
        g.B, g.ldb, g.b_mn_major = self.w_proj_bf.data_ptr(), self.Chid, 1
        g.D, g.ldd = self.dz2.data_ptr(), self.Chid
        if self.se is not None:
            # SE: the GEMM writes d(a2*gate); the gate / pooling gradients need a reduction over
            # HW first, so act'/BN2-backward happen in se_bwd_apply afterwards
            self._call(lib.yamb_pointwise_gemm, g, "pw_project_dgrad",
                       2 * self.M_out * (2 * self.Cout + self.Chid),
                       2 * self.M_out * self.Chid * self.Cout)
            self._se_backward(grads)
        else:
            g.epi = 1
            g.H, g.ldh = self.h2.data_ptr(), self.Chid
            g.h_scale, g.h_shift, g.h_act = self.bn2.scale.data_ptr(), \
                self.bn2.shift.data_ptr(), self.act
            if len(self.bn2.mods) == 1:
                g.bn_bwd = C.pointer(self._bn_bwd_struct(self.bn2, self.M_out, grads["bn2"]))
                self._call(lib.yamb_pointwise_gemm, g, "pw_project_dgrad",
                           4 * self.M_out * (self.Cout + self.Chid),
                           2 * self.M_out * self.Chid * self.Cout)
            else:
                for (c0, cb) in self.bn2.slices:
                    gs = nat.Gemm()
                    C.memmove(C.byref(gs), C.byref(g), C.sizeof(nat.Gemm))
                    gs.N = cb
                    gs.B = g.B + c0 * 2
                    gs.D = g.D + c0 * 2
                    gs.H = g.H + c0 * 2
                    gs.h_scale = g.h_scale + c0 * 4
                    gs.h_shift = g.h_shift + c0 * 4
                    gs.bn_bwd = C.pointer(self._bn_bwd_struct(self.bn2, self.M_out, grads["bn2"],
                                                              c0, cb))
                    self._call(lib.yamb_pointwise_gemm, gs, "pw_project_dgrad",
                               4 * self.M_out * (self.Cout + cb),
                               2 * self.M_out * cb * self.Cout)
        # 3. project wgrad: dW3[Cout,Chid] += dh3^T * a2
        g = nat.Gemm()
        g.M, g.N, g.K = self.Cout, self.Chid, self.M_out
        g.a_mn_major = g.b_mn_major = 1
        g.A, g.lda = dym.data_ptr(), self.Cout
        g.a_xform = 2
        g.a_scale, g.a_scale2, g.a_shift = self.bn3.ca.data_ptr(), self.bn3.cb.data_ptr(), \
            self.bn3.cc.data_ptr()
        g.A2, g.lda2 = self.h3.data_ptr(), self.Cout
        g.B, g.ldb = self.h2.data_ptr(), self.Chid
        g.b_xform, g.b_act = 1, self.act
        g.b_scale, g.b_shift = self.bn2.scale.data_ptr(), self.bn2.shift.data_ptr()
        if self.se is not None:
            g.b_gate, g.gate_rows_per_sample = self.gate.data_ptr(), self.Ho * self.Wo
        g.D, g.ldd = grads["proj"].data_ptr(), self.Chid
        g.epi = 2
        # needs only the BN3-backward coefficients (step 1) -> off the critical chain
        self._call_side(lib.yamb_pointwise_gemm, g, "pw_project_wgrad",
                        2 * self.M_out * (2 * self.Cout + self.Chid),
                        2 * self.M_out * self.Chid * self.Cout, fork_ev, (dy,))
        # 4. depthwise backward per branch
        c0 = 0
        for b, (cb, k) in enumerate(zip(self.channels, self.ks)):
            d = nat.DwBwd()
            d.N, d.H, d.W, d.C, d.ldc, d.k, d.stride = self.N, self.H, self.W, cb, self.Chid, k, \
                self.stride
            d.dz = self.dz2.data_ptr() + c0 * 2
            d.h = self.h2.data_ptr() + c0 * 2
            d.ca = self.bn2.ca.data_ptr() + c0 * 4
            d.cb = self.bn2.cb.data_ptr() + c0 * 4
            d.cc = self.bn2.cc.data_ptr() + c0 * 4
            d.w = self.conv_dw[b].weight.data_ptr()
            d.dw = grads["dw"][b].data_ptr()
            if self.expand:
                d.x = self.h1.data_ptr() + c0 * 2
                d.in_scale = self.bn1.scale.data_ptr() + c0 * 4
                d.in_shift = self.bn1.shift.data_ptr() + c0 * 4
                d.in_act = self.act
                d.dx = self.dz1.data_ptr() + c0 * 2
                d.bn = C.pointer(self._bn_bwd_struct(self.bn1, self.M_in, grads["bn1"], c0, cb))
            else:
                d.x = xm.data_ptr()
                d.dx = dx.data_ptr()
                d.residual = dym_skip.data_ptr() if self.residual else None
            self._call(lib.yamb_depthwise_bwd, d, "dw_bwd", 4 * cb * (self.M_in + self.M_out),
                       4 * self.M_out * cb * k * k)
            c0 += cb
        if not self.expand:
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
        self._call(lib.yamb_pointwise_gemm, g, "pw_expand_dgrad",
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
    """BlockPlan (intermediates + argument structs) of `block` for this input shape.  At most
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


def block_params(block):
    """Parameters of a block in the fixed order the autograd Function receives them."""
    return [p for p in block.parameters()]


class _BlockFn(torch.autograd.Function):
    """autograd boundary of the fused block: forward/backward run the sm_90a kernel sequences.

    Parameter gradients: when a parameter carries a pre-allocated fp32 `.grad` that the flat-arena
    optimizer marked with `_yamb_direct` the kernels accumulate straight into it and autograd gets
    None; otherwise gradients are produced into plan-owned buffers and returned to autograd."""

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
        dx, gmap = run_backward(block, plan, x, dy)
        params = list(block.parameters())
        pgrads = []
        for p in params:
            t = gmap.get(id(p))
            pgrads.append(t.clone() if t is not None else None)
        return (dx, None) + tuple(pgrads)


def run_backward(block, plan, x, dy):
    """Backward kernel sequence of one block; returns dx and {id(param): grad} for the parameters
    whose gradient was NOT accumulated straight into `.grad` (flat-arena direct mode)."""
    if True:
        dy = to_nhwc_bf16(dy)
        params = list(block.parameters())
        direct = all(getattr(p, "_yamb_direct", False) and p.grad is not None for p in params)

        def target(p, zero_buf):
            if direct:
                return p.grad
            zero_buf.zero_()
            return zero_buf

        def bn_targets(bn, key):
            res = []
            if bn is None:
                return res
            for i, m in enumerate(bn.mods):
                if direct:
                    res.append((m.weight.grad, m.bias.grad))
                else:
                    bufs = plan.__dict__.setdefault("_bn_gbuf", {})
                    k2 = (key, i)
                    if k2 not in bufs:
                        bufs[k2] = (torch.zeros_like(m.weight), torch.zeros_like(m.bias))
                    bufs[k2][0].zero_()
                    bufs[k2][1].zero_()
                    res.append(bufs[k2])
            return res

        single_exp = plan.expand and len(plan.conv_exp) == 1
        single_proj = len(plan.conv_proj) == 1
        g = {}
        if plan.expand:
            if single_exp and direct:
                g["exp"] = plan.conv_exp[0].weight.grad.view(plan.Chid, plan.Cin)
            else:
                plan.g_exp.zero_()
                g["exp"] = plan.g_exp
        if single_proj and direct:
            g["proj"] = plan.conv_proj[0].weight.grad.view(plan.Cout, plan.Chid)
        else:
            plan.g_proj.zero_()
            g["proj"] = plan.g_proj
        g["dw"] = [target(c.weight, plan.g_dw[i]) for i, c in enumerate(plan.conv_dw)]
        g["bn1"] = bn_targets(plan.bn1, "bn1")
        g["bn2"] = bn_targets(plan.bn2, "bn2")
        g["bn3"] = bn_targets(plan.bn3, "bn3")
        if plan.se is not None:
            se = plan.se
            g["se"] = {"wr": target(se.se_reduce.weight, plan.g_se["wr"]),
                       "br": target(se.se_reduce.bias, plan.g_se["br"]),
                       "we": target(se.se_expand.weight, plan.g_se["we"]),
                       "be": target(se.se_expand.bias, plan.g_se["be"])}
        if plan.nl is not None:
            g["bn4"] = bn_targets(plan.bn4, "bn4")
            g["nl_dw"] = target(plan.nl.depthwise_conv.weight, plan.g_nl)
        dx = plan.backward(x, dy, g)
        if not (DEFER_JOIN and direct and single_proj and (single_exp or not plan.expand)):
            join_side(plan.dev)   # the gradient hand-over below reads what the wgrads wrote
        # ---- hand gradients to autograd ----
        gmap = {}
        if plan.expand:
            if not (single_exp and direct):
                c0 = 0
                for conv in plan.conv_exp:
                    n = conv.weight.shape[0]
                    piece = plan.g_exp[c0:c0 + n].reshape(conv.weight.shape)
                    if direct:
                        conv.weight.grad.add_(piece)
                    else:
                        gmap[id(conv.weight)] = piece
                    c0 += n
        if not (single_proj and direct):
            c0 = 0
            for conv in plan.conv_proj:
                n = conv.weight.shape[1]
                piece = plan.g_proj[:, c0:c0 + n].reshape(conv.weight.shape)
                if direct:
                    conv.weight.grad.add_(piece)
                else:
                    gmap[id(conv.weight)] = piece
                c0 += n
        if not direct:
            for i, c in enumerate(plan.conv_dw):
                gmap[id(c.weight)] = plan.g_dw[i]
            if plan.nl is not None:
                gmap[id(plan.nl.depthwise_conv.weight)] = plan.g_nl
            for key, bn in (("bn1", plan.bn1), ("bn2", plan.bn2), ("bn3", plan.bn3),
                            ("bn4", getattr(plan, "bn4", None))):
                if bn is None:
                    continue
                for i, m in enumerate(bn.mods):
                    dg, db = g[key][i]
                    gmap[id(m.weight)] = dg
                    gmap[id(m.bias)] = db
        if plan.se is not None and not direct:
            se = plan.se
            for k, prm in (("wr", se.se_reduce.weight), ("br", se.se_reduce.bias),
                           ("we", se.se_expand.weight), ("be", se.se_expand.bias)):
                gmap[id(prm)] = plan.g_se[k]
        return dx, gmap


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
        fused = hasattr(block, "expand_conv")
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
        if fused and hasattr(block.nl_op, "bn"):
            # the non-local norm (output width: never padded) is of the real block's class, which
            # the reference picks from FLAGS.nl_norm at construction time
            import copy
            self.shadow.nl_op.bn = copy.deepcopy(block.nl_op.bn).to(device)
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
        dx, gmap = run_backward(sh.shadow, plan, x, dy)
        grads = sh.gather_grads(gmap, block)
        params = list(block.parameters())
        if all(getattr(p, "_yamb_direct", False) and p.grad is not None for p in params):
            torch._foreach_add_([p.grad for p in params], grads)   # straight into the flat arena
            return (dx, None) + (None,) * len(params)
        return (dx, None) + tuple(grads)


# ------------------------------------------------------------------------------------------------
# Stand-alone BatchNorm + activation behind a convolution torch runs (stem 3x3 / head 1x1
# ConvBNReLU, reference models/mobilenet_base.py:181-203): raw conv output h [N,H,W,C] bf16 ->
# statistics kernel (+ finalize) -> y = act(scale*h + shift); backward: statistics of
# dz = dy*act'(z) (+ finalize: dgamma, dbeta, ca/cb/cc) -> dh = ca*dz + cb*h + cc.
# ------------------------------------------------------------------------------------------------
class _BnActState(Scratch):
    def __init__(self, bn, dev):
        self.bn = _Bn([bn], dev)
        self.ws = Workspace.get(dev)
        self.keep = []
        self.gbuf = None


def _bn_act_state(bn, dev):
    st = bn.__dict__.get("_yamb_bnact")
    if st is None or st.bn.dev != dev:
        st = _BnActState(bn, dev)
        bn.__dict__["_yamb_bnact"] = st
    return st


class _BnActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, h, bn, act, weight, bias):
        lib = nat.lib()
        st = _bn_act_state(bn, h.device)
        st.keep = []
        b = st.bn
        N, Cc, H, W = h.shape
        M = N * H * W
        hm = h.permute(0, 2, 3, 1).reshape(M, Cc)        # view of the channels_last storage
        if b.batch_stats:
            f = nat.BnFwd()
            ws = Workspace.get(h.device)
            f.partials, f.counter = ws.partials.data_ptr(), ws.counter.data_ptr()
            f.gamma, f.beta = nat.ptr(bn.weight), nat.ptr(bn.bias)
            f.eps, f.momentum = b.eps, b.momentum_value()
            if bn.track_running_stats and bn.running_mean is not None:
                f.running_mean, f.running_var = bn.running_mean.data_ptr(), bn.running_var.data_ptr()
                f.num_batches_tracked = nat.ptr(bn.num_batches_tracked)
            f.scale, f.shift = b.scale.data_ptr(), b.shift.data_ptr()
            f.mean, f.invstd = b.mean.data_ptr(), b.invstd.data_ptr()
            f.count = M
            s = nat.BnStats()
            s.M, s.C, s.ldh, s.h, s.bn = M, Cc, Cc, hm.data_ptr(), C.pointer(f)
            st.keep += [f, s]
            launch(lib.yamb_bn_stats_fwd, s, "bn_stats", 2 * M * Cc)
        else:
            with torch.no_grad():
                b.eval_coeffs()
        y = torch.empty_like(h, memory_format=torch.channels_last)
        a = nat.BnApply()
        a.M, a.C, a.ldh, a.ldr, a.ldy = M, Cc, Cc, Cc, Cc
        a.h, a.scale, a.shift, a.act = hm.data_ptr(), b.scale.data_ptr(), b.shift.data_ptr(), act
        a.y = y.data_ptr()
        st.keep.append(a)
        launch(lib.yamb_bn_apply_fwd, a, "bn_apply", 4 * M * Cc)
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
        lib = nat.lib()
        h, coef = ctx.saved_tensors
        bn, act, st = ctx.bn, ctx.act, ctx.st
        b = st.bn
        c_scale, c_shift, c_mean, c_invstd = (coef[i].data_ptr() for i in range(4))
        dy = to_nhwc_bf16(dy)
        N, Cc, H, W = h.shape
        M = N * H * W
        hm = h.permute(0, 2, 3, 1).reshape(M, Cc)
        dym = dy.permute(0, 2, 3, 1).reshape(M, Cc)
        params = [p for p in (bn.weight, bn.bias) if p is not None]
        direct = all(getattr(p, "_yamb_direct", False) and p.grad is not None for p in params)
        if direct:
            dg, db = bn.weight.grad, bn.bias.grad
        else:
            if st.gbuf is None:
                st.gbuf = (torch.zeros_like(bn.weight), torch.zeros_like(bn.bias))
            st.gbuf[0].zero_()
            st.gbuf[1].zero_()
            dg, db = st.gbuf
        g = nat.BnBwd()
        ws = Workspace.get(h.device)
        g.partials, g.counter = ws.partials.data_ptr(), ws.counter.data_ptr()
        g.gamma = nat.ptr(bn.weight)
        g.mean, g.invstd = c_mean, c_invstd
        g.dgamma, g.dbeta = dg.data_ptr(), db.data_ptr()
        g.ca, g.cb, g.cc = b.ca.data_ptr(), b.cb.data_ptr(), b.cc.data_ptr()
        g.count = M
        g.use_batch_stats = 1 if b.batch_stats else 0
        r = nat.BnReduce()
        r.M, r.C, r.lddy, r.ldh = M, Cc, Cc, Cc
        r.dy, r.h, r.bn = dym.data_ptr(), hm.data_ptr(), C.pointer(g)
        r.z_scale, r.z_shift, r.z_act = c_scale, c_shift, act
        launch(lib.yamb_bn_reduce_bwd, r, "bn_reduce", 4 * M * Cc)
        dh = torch.empty_like(h, memory_format=torch.channels_last)
        a = nat.BnBwdApply()
        a.M, a.C, a.lddy, a.ldh, a.lddh = M, Cc, Cc, Cc, Cc
        a.dy, a.h = dym.data_ptr(), hm.data_ptr()
        a.z_scale, a.z_shift, a.z_act = c_scale, c_shift, act
        a.ca, a.cb, a.cc = b.ca.data_ptr(), b.cb.data_ptr(), b.cc.data_ptr()
        a.dh = dh.data_ptr()
        st.keep += [g, r, a]
        launch(lib.yamb_bn_bwd_apply_bwd, a, "bn_bwd_apply", 6 * M * Cc)
        if direct:
            return dh, None, None, None, None
        return dh, None, None, dg.clone(), db.clone()


def bn_act_apply(bn, active_fn, h):
    """y = act(BatchNorm(h)) for a raw convolution output on CUDA (training or eval)."""
    h = to_nhwc_bf16(h)
    if h.shape[1] % 8:
        raise nat.NativeError("bn_act: channel count must be a multiple of 8")
    return _BnActFn.apply(h, bn, act_code_of(active_fn), bn.weight, bn.bias)


# ---- eval mode: the whole block in one launch (csrc/block_eval.cu) ---------------------------------
# YAMB_EVAL_FUSED=0 keeps the four-launch sequence (folded coefficients) for every block.
EVAL_FUSED = os.environ.get("YAMB_EVAL_FUSED", "1") != "0"
EVAL_FUSED_CALLS = 0     # blocks that went through yamb_block_eval_fwd (tests / bench)
# (both eval paths: fused_eval_forward for the unfused class, fused_class_eval_forward for
# InvertedResidualChannelsFused)


def fused_eval_supported(block, x):
    """True when yamb_block_eval_fwd covers this block for this call: no gradient wanted, every
    BatchNorm normalising with running statistics, unfused single-branch block with a 3x3 / 5x5 /
    7x7 depthwise, stride 1 or 2, with or without expansion (reference
    models/mobilenet_base.py:380-421; every block of MobileNetV2-1.0 and of Proxyless-mobile),
    channel counts the kernel's tiles hold."""
    if not EVAL_FUSED or torch.is_grad_enabled() or hasattr(block, "expand_conv"):
        return False
    if block.stride not in (1, 2) or not hasattr(block, "ops"):
        return False
    if len(block.channels) != 1 or list(block.kernel_sizes)[0] not in (3, 5, 7):
        return False
    cin, chid, cout = block.input_dim, block.channels[0], block.output_dim
    if cin % 8 or chid % 8 or cout % 8 or cin > 256 or cout > 320:
        return False
    if not block.expand and chid != cin:
        return False
    if x.dim() != 4 or x.shape[0] * x.shape[2] * x.shape[3] >= 2 ** 30:
        return False
    op = block.ops[0]
    bns = (op[0][1], op[1][1], block.pw_bn) if block.expand else (op[0][1], block.pw_bn)
    for bn in bns:
        if not isinstance(bn, torch.nn.BatchNorm2d) or bn.training or \
                not bn.track_running_stats or bn.running_mean is None:
            return False
    try:
        act = act_code_of(block.active_fn)
    except ValueError:
        return False
    if block.kernel_sizes[0] != 3 and (not block.expand or act not in (0, 1, 2)):
        return False        # k = 5 / 7: built with expansion and relu / relu6 only
    return True


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


def fused_eval_forward(block, x):
    """y = block(x) in eval mode through ONE kernel launch; x channels_last bf16 on CUDA."""
    global EVAL_FUSED_CALLS
    dev = x.device
    N, Cin, H, W = x.shape
    op = block.ops[0]
    if block.expand:
        conv_e, bn1, conv_d, bn2, conv_p = op[0][0], op[0][1], op[1][0], op[1][1], op[2]
    else:
        conv_e, bn1, conv_d, bn2, conv_p = None, None, op[0][0], op[0][1], op[1]
    bn3 = block.pw_bn
    Chid, Cout, stride = block.channels[0], block.output_dim, block.stride
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    w1, w3 = _eval_operands(block, dev, Chid, Cin, Cout, conv_e, conv_p)
    y = torch.empty((N, Cout, Ho, Wo), device=dev, dtype=torch.bfloat16,
                    memory_format=torch.channels_last)
    a = _block_eval_args(block, x, y, w1, w3, conv_d, (bn1, bn2, bn3), block.use_res_connect)
    launch(lib_fn("yamb_block_eval_fwd"), a, "block_eval",
           *_block_eval_cost(block, x, Ho, Wo, block.use_res_connect))
    EVAL_FUSED_CALLS += 1
    return y


# ---- eval mode of InvertedResidualChannelsFused (AutoNL, AtomNAS): the block kernel with the SE
# gate and the non-local tail (reference models/mobilenet_base.py:330-342) ----------------------------
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


def _bn_eval_ready(bn):
    return isinstance(bn, torch.nn.BatchNorm2d) and not bn.training and \
        bn.track_running_stats and bn.running_mean is not None


def _nl_norm_eval_ready(norm):
    """The non-local block's norm is a per-channel affine from running statistics."""
    if isinstance(norm, torch.nn.InstanceNorm2d):
        return _nl_norm_supported(norm) and not norm.training
    return _bn_eval_ready(norm)


def fused_class_eval_supported(block, x):
    """True when the eval path of InvertedResidualChannelsFused covers this block for this call: no
    gradient wanted, every BatchNorm (the non-local block's included, or its tracked InstanceNorm)
    normalising with running statistics, one branch with a 3x3 / 5x5 / 7x7 depthwise (no expansion: 3x3 only), stride 1 or
    2, widths that are multiples of 8 with Cin <= 256 and Cout <= 320, any activation, with or
    without Squeeze-and-Excitation and a non-local block (every block of AutoNL-L, block 1 of
    AtomNAS-C+), minus the shapes FUSED_CLASS_SHAPE_RULE keeps on the four-launch sequence (8
    AutoNL-L blocks take the path with it).  The unfused class has its own rule,
    fused_eval_supported."""
    if not EVAL_FUSED or torch.is_grad_enabled() or not hasattr(block, "expand_conv"):
        return False
    if block.stride not in (1, 2) or len(block.channels) != 1:
        return False
    k = list(block.kernel_sizes)[0]
    cin, chid, cout = block.input_dim, block.channels[0], block.output_dim
    if k not in (3, 5, 7) or cin % 8 or chid % 8 or cout % 8 or cin > 256 or cout > 320:
        return False
    if not block.expand and (k != 3 or chid != cin):
        return False
    if FUSED_CLASS_SHAPE_RULE and (k != 3 or not block.expand):
        return False        # measured slower than the four-launch sequence (see above)
    if x.dim() != 4 or x.shape[0] * x.shape[2] * x.shape[3] >= 2 ** 30:
        return False
    stage = list(block.depth_ops[0].children())[-1]
    bns = [stage[1], block.project_conv[1]] + ([block.expand_conv[1]] if block.expand else [])
    nl = block.nl_op if type(block.nl_op).__name__ != "Identity" else None
    if nl is not None:
        if not _nl_norm_eval_ready(nl.bn):
            return False
        c = int(nl.nl_c * cout)
        if c <= 0 or c % 2 or int(nl.nl_s) < 1:
            return False
    if not all(_bn_eval_ready(bn) for bn in bns):
        return False
    try:
        act_code_of(block.active_fn)
        if hasattr(block.se_op, "se_reduce"):
            act_code_of(block.se_op.active_fn)
    except ValueError:
        return False
    return True


def fused_class_eval_forward(block, x):
    """y = block(x) of an InvertedResidualChannelsFused in eval mode; x channels_last bf16 on CUDA.
    C-ABI calls: the block kernel (1); with SE the pool pass and the gate FCs first (3); with a
    non-local block the kernel writes l = BN3(h3) and the non-local tail follows (+4)."""
    global EVAL_FUSED_CALLS
    dev = x.device
    N, Cin, H, W = x.shape
    conv_e, bn1 = (block.expand_conv[0], block.expand_conv[1]) if block.expand else (None, None)
    stage = list(block.depth_ops[0].children())[-1]
    conv_d, bn2 = stage[0], stage[1]
    conv_p, bn3 = block.project_conv[0], block.project_conv[1]
    Chid, Cout, stride = block.channels[0], block.output_dim, block.stride
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    se = block.se_op if hasattr(block.se_op, "se_reduce") else None
    nl = block.nl_op if type(block.nl_op).__name__ != "Identity" else None
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
    if se is not None:
        # gate = sigmoid(W_e act(W_r mean_HW(a2) + b_r) + b_e): pool pass, then the two FCs
        R = se.se_reduce.weight.shape[0]
        pooled = torch.empty(N, Chid, device=dev, dtype=torch.float32)
        gate = torch.empty(N, Chid, device=dev, dtype=torch.float32)
        uv = torch.empty(2, N, R, device=dev, dtype=torch.float32)
        a.pooled = pooled.data_ptr()
        launch(lib_fn("yamb_block_eval_pool_fwd"), a, "block_eval_pool",
               *_block_eval_cost(block, x, Ho, Wo, False, project=False))
        f = nat.SeFc()
        f.N, f.C, f.R, f.act = N, Chid, R, act_code_of(se.active_fn)
        f.pooled = pooled.data_ptr()
        f.w_r, f.b_r = se.se_reduce.weight.data_ptr(), se.se_reduce.bias.data_ptr()
        f.w_e, f.b_e = se.se_expand.weight.data_ptr(), se.se_expand.bias.data_ptr()
        f.u, f.v, f.gate = uv[0].data_ptr(), uv[1].data_ptr(), gate.data_ptr()
        launch(lib_fn("yamb_se_fc_fwd"), f, "se_fc", 4 * N * Chid * 2, 4 * N * Chid * R)
        a.pooled = None
        a.gate = gate.data_ptr()
    launch(lib_fn("yamb_block_eval_fwd"), a, "block_eval",
           *_block_eval_cost(block, x, Ho, Wo, residual))
    if tail is not None:
        xm = x.permute(0, 2, 3, 1).reshape(N * H * W, Cin)    # view, NHWC matrix
        tail.forward(xm, y.permute(0, 2, 3, 1).reshape(N * Ho * Wo, Cout), block.use_res_connect)
    EVAL_FUSED_CALLS += 1
    return y


def block_apply(block, x):
    """Forward of a reference-compatible block module through the sm_90a path."""
    if not x.is_cuda:
        raise nat.NativeError(
            "the inverted-residual block runs only on CUDA sm_90a (no CPU fallback); got a %s "
            "tensor" % x.device)
    x = to_nhwc_bf16(x)
    if fused_eval_supported(block, x):
        return fused_eval_forward(block, x)
    if fused_class_eval_supported(block, x):
        return fused_class_eval_forward(block, x)
    params = list(block.parameters())
    if needs_padding(block):
        return _PadFn.apply(x, block, *params)
    return _BlockFn.apply(x, block, *params)
