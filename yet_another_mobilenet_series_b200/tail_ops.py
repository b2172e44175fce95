"""The layers around the inverted-residual stack on the sm_90a path (SURVEY.md §8f-2):

  head   ConvBNReLU 1x1 (320 -> 1280)      reference models/mobilenet_supernet.py:152-158
  fc     nn.Linear (1280 -> classes)       reference models/mobilenet_supernet.py:163-167
  loss   CrossEntropyLabelSmooth + top-k   reference utils/optim.py:150-158, common.py:67-80

A 1x1 convolution on NHWC activations and a Linear layer are the same [pixels, Cin] x [Cout, Cin]^T
GEMM the blocks already use (`yamb_pointwise_gemm`, wgmma): forward with the BatchNorm
statistics in the epilogue, dgrad with the weight read MN-major, wgrad as split-K with pixels on
K.  The loss is one kernel forward / one backward (`yamb_softmax_ce_*`).  Round 1 ran all of these
through cuDNN / cuBLAS / ~20 ATen launches.
"""
import ctypes as C

import torch

from . import engine
from . import native as nat


def _mat(t):
    """[N, C, H, W] channels_last -> the [N*H*W, C] row-major matrix it is stored as (a view)."""
    n, c, h, w = t.shape
    return t.permute(0, 2, 3, 1).reshape(n * h * w, c)


class _PwState(engine.Scratch):
    """Per-module device state of a 1x1 convolution: bf16 weight copy."""

    def __init__(self, conv, dev):
        self.w_own = torch.empty(conv.out_channels, conv.in_channels, device=dev,
                                 dtype=torch.bfloat16)
        self.dev = dev


def _pw_state(conv, dev):
    st = conv.__dict__.get("_yamb_pw")
    if st is None or st.dev != dev:
        st = conv.__dict__["_yamb_pw"] = _PwState(conv, dev)
    return st


def _gemm(M, N, K, A, lda, B, ldb, D, ldd, **kw):
    g = nat.Gemm()
    g.M, g.N, g.K = M, N, K
    g.A, g.lda, g.B, g.ldb, g.D, g.ldd = A, lda, B, ldb, D, ldd
    for k, v in kw.items():
        setattr(g, k, v)
    return g


class _PwConvFn(torch.autograd.Function):
    """Raw output h = conv1x1(x) of a ConvBNReLU by the GEMM, which takes the batch statistics of
    the BatchNorm `bn` behind it in its epilogue when `bn` normalises with them; backward: dgrad
    GEMM + split-K wgrad GEMM."""

    @staticmethod
    def forward(ctx, x, conv, bn, weight):
        st = _pw_state(conv, x.device)
        N, Cin, H, W = x.shape
        Cout = conv.out_channels
        M = N * H * W
        with torch.no_grad():
            wbf = engine._bf16_operand(conv.weight, st.w_own, (Cout, Cin))
        h = torch.empty((N, Cout, H, W), device=x.device, dtype=torch.bfloat16,
                        memory_format=torch.channels_last)
        g = _gemm(M, Cout, Cin, _mat(x).data_ptr(), Cin, wbf.data_ptr(), Cin, h.data_ptr(), Cout)
        b = engine._bn_act_state(bn, x.device).bn
        if b.batch_stats:
            g.bn_fwd = C.pointer(b.fwd_struct(M))
        engine.launch(nat.lib().yamb_pointwise_gemm, g, "head_conv_fwd", 2 * M * (Cin + Cout),
                      2 * M * Cin * Cout)
        ctx.conv = conv
        ctx.save_for_backward(x, wbf)
        return h

    @staticmethod
    def backward(ctx, dh):
        lib = nat.lib()
        x, wbf = ctx.saved_tensors
        conv = ctx.conv
        dh = engine.to_nhwc_bf16(dh)
        N, Cin, H, W = x.shape
        Cout = conv.out_channels
        M = N * H * W
        gt = engine.GradTargets((conv.weight,))
        gw = gt.of(conv.weight)
        # dgrad: dx[M, Cin] = dh[M, Cout] * W[Cout, Cin]   (weight read MN-major)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty((N, Cin, H, W), device=x.device, dtype=torch.bfloat16,
                             memory_format=torch.channels_last)
            g = _gemm(M, Cin, Cout, dh.data_ptr(), Cout, wbf.data_ptr(), Cin, dx.data_ptr(), Cin,
                      b_mn_major=1)
            engine.launch(lib.yamb_pointwise_gemm, g, "head_conv_dgrad", 2 * M * (Cin + Cout),
                          2 * M * Cin * Cout)
        # wgrad: dW[Cout, Cin] += dh^T x   (pixels on K, split-K, slabs added in a fixed order)
        g2 = _gemm(Cout, Cin, M, dh.data_ptr(), Cout, _mat(x).data_ptr(), Cin, gw.data_ptr(), Cin,
                   a_mn_major=1, b_mn_major=1, epi=2)
        engine.launch(lib.yamb_pointwise_gemm, g2, "head_conv_wgrad", 2 * M * (Cin + Cout),
                      2 * M * Cin * Cout)
        return (dx, None, None) + gt.result()


def pw_conv_bn_act(mod, x):
    """ConvBNReLU with a 1x1 convolution (reference models/mobilenet_base.py:181-203) on CUDA:
    pointwise GEMM (+ BatchNorm statistics in its epilogue) -> BatchNorm apply + activation
    (engine.bn_act_apply)."""
    x = engine.to_nhwc_bf16(x)
    conv, bn, act = mod[0], mod[1], mod[2]
    h = _PwConvFn.apply(x, conv, bn, conv.weight)
    return engine.bn_act_apply(bn, act, h, stats_taken=True)


def _tail_eval_wanted(bn):
    return engine.EVAL_TAIL_FUSED and not torch.is_grad_enabled() and engine._bn_eval_ready(bn)


def head_pool_eval(mod, x):
    """Eval-mode head ConvBNReLU 1x1 followed by the full-extent average pool in one launch
    (yamb_head_pool_eval_fwd): bf16 [N, Cout, 1, 1], or None when the call is not covered
    (switch off, gradient wanted, BatchNorm on batch statistics, shape) and the caller runs the
    unfused sequence."""
    conv, bn, act = mod[0], mod[1], mod[2]
    if not (_tail_eval_wanted(bn) and pw_conv_supported(mod, x)):
        return None
    x = engine.to_nhwc_bf16(x)
    N, Cin, H, W = x.shape
    Cout = conv.out_channels
    st = _pw_state(conv, x.device)
    b = engine._bn_act_state(bn, x.device).bn
    with torch.no_grad():
        wbf = engine._bf16_operand(conv.weight, st.w_own, (Cout, Cin))
        b.eval_coeffs()
    pooled = torch.empty(N, Cout, device=x.device, dtype=torch.bfloat16)
    a = nat.HeadPoolEval()
    a.N, a.HW, a.Cin, a.Cout = N, H * W, Cin, Cout
    a.x, a.w = x.data_ptr(), wbf.data_ptr()
    a.scale, a.shift, a.act = b.scale.data_ptr(), b.shift.data_ptr(), engine.act_code_of(act)
    a.pooled = pooled.data_ptr()
    if not engine.try_launch(nat.lib().yamb_head_pool_eval_fwd, a, "head_pool_eval",
                             2 * (N * H * W * Cin + Cout * Cin + N * Cout), 2 * N * H * W * Cin * Cout):
        return None
    engine.EVAL_TAIL_CALLS += 1
    return pooled.view(N, Cout, 1, 1)


class _HeadPoolTrainFn(torch.autograd.Function):
    """pooled[N, C] = the pixel mean of act(BatchNorm(h)), BatchNorm on the batch statistics the
    head GEMM's epilogue took (yamb_head_pool_train_fwd); backward: dh from dpooled in two passes
    (yamb_head_pool_train_bwd), dgamma / dbeta through engine.GradTargets."""

    @staticmethod
    def forward(ctx, h, bn, act, weight, bias):
        b = engine._bn_act_state(bn, h.device).bn
        N, Cc, H, W = h.shape
        pooled = torch.empty(N, Cc, device=h.device, dtype=torch.bfloat16)
        a = nat.HeadPoolTrain()
        a.N, a.HW, a.C = N, H * W, Cc
        a.h, a.scale, a.shift, a.act = h.data_ptr(), b.scale.data_ptr(), b.shift.data_ptr(), act
        a.pooled = pooled.data_ptr()
        engine.launch(nat.lib().yamb_head_pool_train_fwd, a, "head_pool_train",
                      2 * N * Cc * (H * W + 1))
        ctx.bn, ctx.act = bn, act
        # this call's coefficients, as _BnActFn keeps them (another forward through the module
        # before this backward, e.g. the next micro-batch, rewrites the live ones)
        coef = torch.stack((b.scale, b.shift, b.mean, b.invstd)) if any(ctx.needs_input_grad) \
            else None
        ctx.save_for_backward(h, coef)
        return pooled

    @staticmethod
    def backward(ctx, dpooled):
        h, coef = ctx.saved_tensors
        bn = ctx.bn
        b = engine._bn_act_state(bn, h.device).bn
        N, Cc, H, W = h.shape
        M = N * H * W
        dpooled = dpooled.to(torch.bfloat16).contiguous()
        gt = engine.GradTargets((bn.weight, bn.bias))
        g = nat.HeadPoolTrainGrad()
        g.N, g.HW, g.C = N, H * W, Cc
        g.h, g.act = h.data_ptr(), ctx.act
        g.scale, g.shift = coef[0].data_ptr(), coef[1].data_ptr()
        g.dpooled = dpooled.data_ptr()
        g.bn = b.bwd_struct(M, [(gt.of(bn.weight), gt.of(bn.bias))])
        g.bn.mean, g.bn.invstd = coef[2].data_ptr(), coef[3].data_ptr()
        dh = None
        if ctx.needs_input_grad[0]:
            dh = torch.empty_like(h, memory_format=torch.channels_last)
            g.dh = dh.data_ptr()
        engine.launch(nat.lib().yamb_head_pool_train_bwd, g, "head_pool_train_bwd",
                      2 * M * Cc * (3 if dh is not None else 1))
        return (dh, None, None) + gt.result()


def head_pool_train_covered(mod, x):
    """Whether head_pool_train runs ConvBNReLU `mod` on x: engine.TRAIN_TAIL_FUSED is on, the
    BatchNorm normalises with batch statistics and the GEMM and the kernels cover the layer (the
    caller checks that an average pool over the whole map follows)."""
    bn = mod[1]
    return (engine.TRAIN_TAIL_FUSED and (bn.training or not bn.track_running_stats)
            and pw_conv_supported(mod, x))


def head_pool_train(mod, x):
    """Training-mode head ConvBNReLU 1x1 followed by the full-extent average pool: the head GEMM
    (BatchNorm statistics in its epilogue) -> yamb_head_pool_train_fwd, bf16 [N, Cout, 1, 1]; or
    None when the call is not covered (head_pool_train_covered) and the caller runs the unfused
    sequence."""
    if not head_pool_train_covered(mod, x):
        return None
    x = engine.to_nhwc_bf16(x)
    conv, bn, act = mod[0], mod[1], mod[2]
    h = _PwConvFn.apply(x, conv, bn, conv.weight)
    pooled = _HeadPoolTrainFn.apply(h, bn, engine.act_code_of(act), bn.weight, bn.bias)
    engine.TRAIN_TAIL_CALLS += 1
    return pooled.view(pooled.shape[0], pooled.shape[1], 1, 1)


def pw_conv_supported(mod, x):
    conv, bn, act = mod[0], mod[1], mod[2]
    return (x.is_cuda and conv.kernel_size == (1, 1) and conv.stride == (1, 1) and conv.groups == 1
            and conv.bias is None and conv.in_channels % 8 == 0 and conv.out_channels % 8 == 0
            and bn.affine and type(act).__name__ in ("ReLU", "ReLU6", "Swish", "HSwish", "Identity"))


# ---- classifier --------------------------------------------------------------------------------
class _LinearState(engine.Scratch):
    def __init__(self, lin, dev):
        self.w_own = torch.empty(lin.out_features, lin.in_features, device=dev,
                                 dtype=torch.bfloat16)
        self.bias_bf = torch.empty(lin.out_features, device=dev, dtype=torch.bfloat16)
        self.dev = dev


class _LinearFn(torch.autograd.Function):
    """logits[M, O] = x[M, I] W[O, I]^T + bias (bf16 operands, fp32 accumulation, bf16 logits)."""

    @staticmethod
    def forward(ctx, x, lin, weight, bias):
        lib = nat.lib()
        st = lin.__dict__.get("_yamb_lin")
        if st is None or st.dev != x.device:
            st = _LinearState(lin, x.device)
            lin.__dict__["_yamb_lin"] = st
        M, I = x.shape
        O = lin.out_features
        with torch.no_grad():
            wbf = engine._bf16_operand(lin.weight, st.w_own, (O, I))
            st.bias_bf.copy_(lin.bias)
        y = torch.empty(M, O, device=x.device, dtype=torch.bfloat16)
        # the bias enters as a "residual" whose row pitch is 0: every output row adds the same row
        g = _gemm(M, O, I, x.data_ptr(), I, wbf.data_ptr(), I, y.data_ptr(), O,
                  residual=st.bias_bf.data_ptr(), ldr=0)
        engine.launch(lib.yamb_pointwise_gemm, g, "fc_fwd", 2 * (M * I + O * I + M * O),
                      2 * M * I * O)
        ctx.lin = lin
        ctx.save_for_backward(x, wbf)
        return y

    @staticmethod
    def backward(ctx, dy):
        lib = nat.lib()
        x, wbf = ctx.saved_tensors
        lin = ctx.lin
        M, I = x.shape
        O = lin.out_features
        dy = dy.contiguous()
        if dy.dtype != torch.bfloat16:
            dy = dy.to(torch.bfloat16)
        gt = engine.GradTargets((lin.weight, lin.bias))
        gw = gt.of(lin.weight)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty(M, I, device=x.device, dtype=torch.bfloat16)
            g = _gemm(M, I, O, dy.data_ptr(), O, wbf.data_ptr(), I, dx.data_ptr(), I, b_mn_major=1)
            engine.launch(lib.yamb_pointwise_gemm, g, "fc_dgrad", 2 * (M * I + O * I + M * O),
                          2 * M * I * O)
        g2 = _gemm(O, I, M, dy.data_ptr(), O, x.data_ptr(), I, gw.data_ptr(), I,
                   a_mn_major=1, b_mn_major=1, epi=2)
        engine.launch(lib.yamb_pointwise_gemm, g2, "fc_wgrad", 2 * (M * I + M * O) + 4 * O * I,
                      2 * M * I * O)
        # bias gradient: column sums of dlogits
        nat.check(lib.yamb_colsum_bf16(dy.data_ptr(), M, O, O, gt.of(lin.bias).data_ptr(),
                                       nat.stream_handle()))
        engine.LAUNCHES += 1
        return (dx, None) + gt.result()


def linear_apply(lin, x):
    """nn.Linear on CUDA through the wgmma GEMM (in/out features multiples of 8)."""
    if x.dtype != torch.bfloat16 or not x.is_contiguous():
        x = x.to(torch.bfloat16).contiguous()
    return _LinearFn.apply(x, lin, lin.weight, lin.bias)


def linear_supported(lin, x):
    return (x.is_cuda and x.dim() == 2 and lin.bias is not None and lin.in_features % 8 == 0
            and lin.out_features % 8 == 0)


# ---- loss --------------------------------------------------------------------------------------
class _SoftmaxCeFn(torch.autograd.Function):
    """Per-sample label-smoothed cross entropy (reference CrossEntropyLabelSmooth with
    reduction='none', utils/optim.py:150-158) + the top-1 / top-5 indicators of common.py:73-79."""

    @staticmethod
    def forward(ctx, logits, target, smoothing):
        lib = nat.lib()
        if logits.dtype != torch.bfloat16 or not logits.is_contiguous():
            logits = logits.to(torch.bfloat16).contiguous()
        N, Cc = logits.shape
        dev = logits.device
        loss = torch.empty(N, device=dev, dtype=torch.float32)
        c1 = torch.empty(N, device=dev, dtype=torch.float32)
        c5 = torch.empty(N, device=dev, dtype=torch.float32)
        G = torch.empty(N, Cc, device=dev, dtype=torch.bfloat16) if ctx.needs_input_grad[0] \
            else None
        a = nat.SoftmaxCe()
        a.N, a.C, a.ld = N, Cc, Cc
        a.logits, a.target = logits.data_ptr(), target.data_ptr()
        a.smoothing = float(smoothing)
        a.loss, a.correct1, a.correct5 = loss.data_ptr(), c1.data_ptr(), c5.data_ptr()
        a.G, a.ldg = nat.ptr(G), Cc
        engine.launch(lib.yamb_softmax_ce_fwd, a, "softmax_ce", 4 * N * Cc)
        ctx.save_for_backward(G)
        ctx.mark_non_differentiable(c1, c5)
        return loss, c1, c5

    @staticmethod
    def backward(ctx, dloss, _d1, _d5):
        lib = nat.lib()
        (G,) = ctx.saved_tensors
        N, Cc = G.shape
        dloss = dloss.contiguous().float()
        dl = torch.empty(N, Cc, device=G.device, dtype=torch.bfloat16)
        a = nat.SoftmaxCeGrad()
        a.N, a.C = N, Cc
        a.G, a.ldg = G.data_ptr(), Cc
        a.dloss = dloss.data_ptr()
        a.dlogits, a.ldd = dl.data_ptr(), Cc
        engine.launch(lib.yamb_softmax_ce_bwd, a, "softmax_ce_bwd", 4 * N * Cc)
        return dl, None, None


def softmax_ce(logits, target, smoothing):
    """(per-sample loss [N] fp32, correct@1 [N], correct@5 [N]) of bf16/fp32 logits on CUDA."""
    if not logits.is_cuda:
        raise nat.NativeError("softmax_ce runs only on CUDA (no CPU fallback)")
    if target.dtype != torch.long:
        target = target.long()
    return _SoftmaxCeFn.apply(logits, target.contiguous(), smoothing)


# ---- stem ----------------------------------------------------------------------------------------
# `norm` = ((mean x 3), (std x 3)) marks a uint8 image: x is uint8 [N, 3, H, W] channels_last, and
# the yamb_stem_conv_u8_* entries normalise it inside the kernels, with the bits of torchvision's
# ToTensor() + Normalize() on the host followed by the bf16 cast (no normalised tensor in HBM).
def _stem_args(norm, eval_args=False):
    """(argument struct, its yamb_stem_conv part, its yamb_stem_conv_eval part or None) of a call
    on a bf16 x (`norm` None) or a uint8 x."""
    if norm is None:
        if eval_args:
            a = nat.StemConvEval()
            return a, a.conv, a
        a = nat.StemConv()
        return a, a, None
    a = nat.StemConvU8()
    a.mean[:] = norm[0]
    a.std[:] = norm[1]
    return a, a.ev.conv, a.ev


def _stem_bytes(x, Ho, Wo, Cout):
    N, _, H, W = x.shape
    return N * (H * W * 3 * x.element_size() + 2 * Ho * Wo * Cout)


class _StemConvFn(torch.autograd.Function):
    """Raw output of the 3x3 / stride-2 / 3-channel first convolution (reference
    models/mobilenet_supernet.py:124-130) by the direct kernels of csrc/stem.cu; weight gradient
    in backward, no input gradient."""

    @staticmethod
    def forward(ctx, x, conv, norm, weight):
        lib = nat.lib()
        N, _, H, W = x.shape
        Cout = conv.out_channels
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        y = torch.empty((N, Cout, Ho, Wo), device=x.device, dtype=torch.bfloat16,
                        memory_format=torch.channels_last)
        a, c, _ = _stem_args(norm)
        c.N, c.H, c.W, c.Cout = N, H, W, Cout
        c.x, c.w, c.y = x.data_ptr(), conv.weight.data_ptr(), y.data_ptr()
        if norm is None:
            engine.launch(lib.yamb_stem_conv_fwd, a, "stem_conv_fwd",
                          _stem_bytes(x, Ho, Wo, Cout), 2 * N * Ho * Wo * Cout * 27)
        else:
            engine.launch(lib.yamb_stem_conv_u8_fwd, a, "stem_conv_u8_fwd",
                          _stem_bytes(x, Ho, Wo, Cout), 2 * N * Ho * Wo * Cout * 27)
        ctx.conv = conv
        ctx.norm = norm
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, dh):
        lib = nat.lib()
        (x,) = ctx.saved_tensors
        conv = ctx.conv
        dh = engine.to_nhwc_bf16(dh)
        N, _, H, W = x.shape
        Cout = conv.out_channels
        gt = engine.GradTargets((conv.weight,))
        a, c, _ = _stem_args(ctx.norm)
        c.N, c.H, c.W, c.Cout = N, H, W, Cout
        c.x, c.dh, c.dw = x.data_ptr(), dh.data_ptr(), gt.of(conv.weight).data_ptr()
        Ho, Wo = dh.shape[2], dh.shape[3]
        if ctx.norm is None:
            engine.launch(lib.yamb_stem_conv_wgrad, a, "stem_conv_wgrad",
                          _stem_bytes(x, Ho, Wo, Cout), 2 * N * Ho * Wo * Cout * 27)
        else:
            engine.launch(lib.yamb_stem_conv_u8_wgrad, a, "stem_conv_u8_wgrad",
                          _stem_bytes(x, Ho, Wo, Cout), 2 * N * Ho * Wo * Cout * 27)
        return (None, None, None) + gt.result()


def stem_supported(mod, x):
    conv, bn, act = mod[0], mod[1], mod[2]
    co = conv.out_channels
    return (x.is_cuda and conv.in_channels == 3 and conv.kernel_size == (3, 3)
            and conv.stride == (2, 2) and conv.padding == (1, 1) and conv.groups == 1
            and conv.dilation == (1, 1) and conv.bias is None and co in (8, 16, 32, 64)
            and bn.affine
            and type(act).__name__ in ("ReLU", "ReLU6", "Swish", "HSwish", "Identity"))


def stem_conv_bn_act(mod, x, norm=None):
    """ConvBNReLU(3, C, stride=2) on CUDA: direct convolution kernel -> BatchNorm statistics ->
    BatchNorm apply + activation (engine.bn_act_apply).  With `norm`, x is a uint8 image the
    kernels normalise."""
    if norm is None:
        x = engine.to_nhwc_bf16(x)
    conv, bn, act = mod[0], mod[1], mod[2]
    if _tail_eval_wanted(bn):
        y = _stem_eval(conv, bn, act, x, norm)
        if y is not None:
            return y
    h = _StemConvFn.apply(x, conv, norm, conv.weight)
    return engine.bn_act_apply(bn, act, h)


def _stem_eval(conv, bn, act, x, norm=None):
    """Eval-mode stem in one launch (yamb_stem_conv_eval_fwd, or yamb_stem_conv_u8_eval_fwd on a
    uint8 x), bitwise equal to the stem kernel followed by bn_act_apply; None when the kernel
    declines the shape."""
    N, _, H, W = x.shape
    Cout = conv.out_channels
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    b = engine._bn_act_state(bn, x.device).bn
    with torch.no_grad():
        b.eval_coeffs()
    y = torch.empty((N, Cout, Ho, Wo), device=x.device, dtype=torch.bfloat16,
                    memory_format=torch.channels_last)
    a, c, e = _stem_args(norm, eval_args=True)
    c.N, c.H, c.W, c.Cout = N, H, W, Cout
    c.x, c.w, c.y = x.data_ptr(), conv.weight.data_ptr(), y.data_ptr()
    e.scale, e.shift, e.act = b.scale.data_ptr(), b.shift.data_ptr(), engine.act_code_of(act)
    fn = nat.lib().yamb_stem_conv_eval_fwd if norm is None else nat.lib().yamb_stem_conv_u8_eval_fwd
    if not engine.try_launch(fn, a, "stem_conv_eval", _stem_bytes(x, Ho, Wo, Cout),
                             2 * N * Ho * Wo * Cout * 27):
        return None
    engine.EVAL_TAIL_CALLS += 1
    return y


_NORM_TENSORS = {}


def normalize_u8(x, norm):
    """uint8 [N, 3, H, W] -> bf16 channels_last ((x / 255 - mean) / std), with the fp32 operations
    and rounding of torchvision's ToTensor() + Normalize() on the host, then the bf16 cast: the
    input of a stem the direct kernels do not cover.  Every divisor is a device tensor: CUDA torch
    may turn a division by a Python scalar into a multiply by its reciprocal, other bits."""
    key = (norm, x.device)
    t = _NORM_TENSORS.get(key)
    if t is None:       # built on the first (eager) call, so a graph capture later copies nothing
        mk = lambda v: torch.tensor(v, dtype=torch.float32, device=x.device).view(1, 3, 1, 1)
        t = _NORM_TENSORS[key] = (mk((255.0,) * 3), mk(norm[0]), mk(norm[1]))
    y = x.float().div_(t[0]).sub_(t[1]).div_(t[2])
    return y.to(dtype=torch.bfloat16, memory_format=torch.channels_last)


def stem_u8(mod, x, norm):
    """The first layer of a network fed a uint8 image `x` (channels_last) with normalisation
    `norm`: the uint8 stem kernels when they cover the layer, else the layer on the image
    normalised on the device (normalize_u8)."""
    if isinstance(mod, torch.nn.Sequential) and len(mod) == 3 and stem_supported(mod, x):
        return stem_conv_bn_act(mod, x, norm)
    return mod(normalize_u8(x, norm))


# ---- training mode: the stem and its only consumer ----------------------------------------------
def stem_block_fused_covered(stem, block, x):
    """Whether stem_block_train runs the stem ConvBNReLU `stem` on image x together with the next
    layer `block`: the direct stem kernels cover the stem, its BatchNorm normalises with batch
    statistics, `block` is an inverted-residual block (either class, with or without SE or
    non-local) without expansion, with one branch and no skip connection, whose input width is the
    stem's output width, and that runs on the training path (not engine.eval_forward).  Then the
    block's depthwise is the only reader of the stem activation.  Host-only: reads shapes and
    modules, no device."""
    from .mobilenet_base import _FusedBlockBase
    if not (isinstance(stem, torch.nn.Sequential) and len(stem) == 3 and stem_supported(stem, x)):
        return False
    bn = stem[1]
    if not (isinstance(bn, torch.nn.BatchNorm2d) and (bn.training or not bn.track_running_stats)):
        return False
    cout = stem[0].out_channels
    if not (isinstance(block, _FusedBlockBase) and not block.expand and len(block.channels) == 1
            and not block.use_res_connect and block.input_dim == cout
            and block.channels[0] == cout):
        return False
    N, _, H, W = x.shape
    h = torch.empty((N, cout, (H - 1) // 2 + 1, (W - 1) // 2 + 1), device="meta")
    return not engine.eval_supported(block, h)


def _stem_train_args(st, x, conv, norm):
    st.N, st.H, st.W, st.Cout = x.shape[0], x.shape[2], x.shape[3], conv.out_channels
    st.x = x.data_ptr()
    if norm is not None:
        st.x_u8 = 1
        st.mean[:] = norm[0]
        st.std[:] = norm[1]


class _StemBlockFn(torch.autograd.Function):
    """Stem ConvBNReLU + the first block (stem_block_fused_covered) as one autograd function.
    Forward: yamb_stem_conv_train_fwd writes the raw stem output h and finalises the stem
    BatchNorm's batch statistics; the block's BlockPlan runs with the stem's BatchNorm +
    activation applied by its depthwise on load.  Backward: the BlockPlan backward, whose
    depthwise writes dz_stem = da * act'(z) and the stem BatchNorm's backward statistics
    (dgamma, dbeta, ca / cb / cc), then yamb_stem_conv_train_wgrad forms dh on load.  Gradients
    of the stem weight, the stem BatchNorm and the block go through engine.GradTargets."""

    @staticmethod
    def forward(ctx, x, stem, block, norm, *params):
        lib = nat.lib()
        conv, bn = stem[0], stem[1]
        act = engine.act_code_of(stem[2])
        b = engine._bn_act_state(bn, x.device).bn
        N, _, H, W = x.shape
        Cout = conv.out_channels
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        h = torch.empty((N, Cout, Ho, Wo), device=x.device, dtype=torch.bfloat16,
                        memory_format=torch.channels_last)
        a = nat.StemConvTrain()
        _stem_train_args(a, x, conv, norm)
        a.w, a.y = conv.weight.data_ptr(), h.data_ptr()
        stats = b.fwd_struct(N * Ho * Wo)
        a.bn = C.pointer(stats)
        engine.launch(lib.yamb_stem_conv_train_fwd, a, "stem_conv_train_fwd",
                      _stem_bytes(x, Ho, Wo, Cout), 2 * N * Ho * Wo * Cout * 27)
        # this call's coefficients, as _BnActFn keeps them (another forward through the stem
        # before this backward, e.g. the next micro-batch, rewrites the live ones)
        coef = torch.stack((b.scale, b.shift, b.mean, b.invstd))
        plan = engine._plan_for(block, h)
        y = plan.forward(h, pre=(coef[0], coef[1], act))
        ctx.stem, ctx.block, ctx.norm, ctx.act = stem, block, norm, act
        ctx.plan, ctx.generation = plan, plan.generation
        ctx.save_for_backward(x, h, coef)
        return y

    @staticmethod
    def backward(ctx, dy):
        plan = ctx.plan
        if plan.generation != ctx.generation:
            raise RuntimeError("yamb: the first block ran another forward before the backward of "
                               "the previous one (see engine._BlockFn)")
        x, h, coef = ctx.saved_tensors
        conv, bn = ctx.stem[0], ctx.stem[1]
        b = engine._bn_act_state(bn, h.device).bn
        N, Cout, Ho, Wo = h.shape
        dy = engine.to_nhwc_bf16(dy)
        gt = engine.GradTargets([conv.weight, bn.weight, bn.bias] + list(ctx.block.parameters()))
        stats = b.bwd_struct(N * Ho * Wo, [(gt.of(bn.weight), gt.of(bn.bias))])
        stats.mean, stats.invstd = coef[2].data_ptr(), coef[3].data_ptr()
        dz = plan.backward(h, dy, engine.block_grads(gt, plan), pre=(coef[0], coef[1], ctx.act),
                           pre_stats=stats)
        a = nat.StemConvTrainGrad()
        _stem_train_args(a, x, conv, ctx.norm)
        a.dz, a.h = dz.data_ptr(), h.data_ptr()
        a.ca, a.cb, a.cc = b.ca.data_ptr(), b.cb.data_ptr(), b.cc.data_ptr()
        a.dw = gt.of(conv.weight).data_ptr()
        engine.launch(nat.lib().yamb_stem_conv_train_wgrad, a, "stem_conv_train_wgrad",
                      _stem_bytes(x, Ho, Wo, Cout) + 2 * N * Ho * Wo * Cout,
                      2 * N * Ho * Wo * Cout * 27)
        if not engine.DEFER_JOIN or gt.host_reads:
            engine.join_side(plan.dev)
        return (None, None, None, None) + gt.result()


def stem_block_train(stem, block, x, norm=None):
    """y = block(stem(x)) in training through _StemBlockFn, for a pair stem_block_fused_covered
    accepts (the caller checks).  x: bf16 channels_last, or with `norm` a uint8 image the
    kernels normalise."""
    params = [stem[0].weight, stem[1].weight, stem[1].bias] + list(block.parameters())
    y = _StemBlockFn.apply(x, stem, block, norm, *params)
    engine.TRAIN_STEM_CALLS += 1
    return y
