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
    """Per-module device state of a 1x1 ConvBNReLU: BatchNorm coefficients, bf16 weight copy."""

    def __init__(self, conv, bn, dev):
        self.bn = engine._Bn([bn], dev)
        self.ws = engine.Workspace.get(dev)
        self.w_own = torch.empty(conv.out_channels, conv.in_channels, device=dev,
                                 dtype=torch.bfloat16)
        self.g_own = None
        self.gbuf = None
        self.keep = []
        self.dev = dev


def _pw_state(mod, dev):
    st = mod.__dict__.get("_yamb_pw")
    if st is None or st.dev != dev:
        st = _PwState(mod[0], mod[1], dev)
        mod.__dict__["_yamb_pw"] = st
    return st


def _gemm(M, N, K, A, lda, B, ldb, D, ldd, **kw):
    g = nat.Gemm()
    g.M, g.N, g.K = M, N, K
    g.A, g.lda, g.B, g.ldb, g.D, g.ldd = A, lda, B, ldb, D, ldd
    for k, v in kw.items():
        setattr(g, k, v)
    return g


class _PwConvBnActFn(torch.autograd.Function):
    """y = act(BatchNorm(conv1x1(x))) — GEMM (+ statistics) -> BN apply; backward: BN-backward
    reduction -> dh -> dgrad GEMM + split-K wgrad GEMM."""

    @staticmethod
    def forward(ctx, x, mod, act, weight, gamma, beta):
        lib = nat.lib()
        conv, bn = mod[0], mod[1]
        st = _pw_state(mod, x.device)
        st.keep = []
        b = st.bn
        N, Cin, H, W = x.shape
        Cout = conv.out_channels
        M = N * H * W
        xm = _mat(x)
        with torch.no_grad():
            wbf = engine._bf16_operand(conv.weight, st.w_own, (Cout, Cin))
        h = torch.empty((N, Cout, H, W), device=x.device, dtype=torch.bfloat16,
                        memory_format=torch.channels_last)
        g = _gemm(M, Cout, Cin, xm.data_ptr(), Cin, wbf.data_ptr(), Cin, h.data_ptr(), Cout)
        if b.batch_stats:
            f = nat.BnFwd()
            ws = engine.Workspace.get(x.device)
            f.partials, f.counter = ws.partials.data_ptr(), ws.counter.data_ptr()
            f.gamma, f.beta = nat.ptr(bn.weight), nat.ptr(bn.bias)
            f.eps, f.momentum = b.eps, b.momentum_value()
            if bn.track_running_stats and bn.running_mean is not None:
                f.running_mean, f.running_var = bn.running_mean.data_ptr(), \
                    bn.running_var.data_ptr()
                f.num_batches_tracked = nat.ptr(bn.num_batches_tracked)
            f.scale, f.shift = b.scale.data_ptr(), b.shift.data_ptr()
            f.mean, f.invstd = b.mean.data_ptr(), b.invstd.data_ptr()
            f.count = M
            g.bn_fwd = C.pointer(f)
            st.keep.append(f)
        else:
            with torch.no_grad():
                b.eval_coeffs()
        st.keep.append(g)
        engine.launch(lib.yamb_pointwise_gemm, g, "head_conv_fwd", 2 * M * (Cin + Cout),
                      2 * M * Cin * Cout)
        y = torch.empty_like(h, memory_format=torch.channels_last)
        a = nat.BnApply()
        a.M, a.C, a.ldh, a.ldr, a.ldy = M, Cout, Cout, Cout, Cout
        a.h, a.scale, a.shift, a.act = h.data_ptr(), b.scale.data_ptr(), b.shift.data_ptr(), act
        a.y = y.data_ptr()
        st.keep.append(a)
        engine.launch(lib.yamb_bn_apply_fwd, a, "bn_apply", 4 * M * Cout)
        coef = torch.stack((b.scale, b.shift, b.mean, b.invstd)) if any(ctx.needs_input_grad) \
            else None
        ctx.mod, ctx.act, ctx.st = mod, act, st
        ctx.save_for_backward(x, h, coef, wbf)
        return y

    @staticmethod
    def backward(ctx, dy):
        lib = nat.lib()
        x, h, coef, wbf = ctx.saved_tensors
        mod, act, st = ctx.mod, ctx.act, ctx.st
        conv, bn = mod[0], mod[1]
        b = st.bn
        dy = engine.to_nhwc_bf16(dy)
        N, Cin, H, W = x.shape
        Cout = conv.out_channels
        M = N * H * W
        xm, hm, dym = _mat(x), _mat(h), _mat(dy)
        c_scale, c_shift, c_mean, c_invstd = (coef[i].data_ptr() for i in range(4))
        params = [conv.weight, bn.weight, bn.bias]
        direct = all(getattr(p, "_yamb_direct", False) and p.grad is not None for p in params)
        if direct:
            dg, db, gw = bn.weight.grad, bn.bias.grad, conv.weight.grad
        else:
            if st.gbuf is None:
                st.gbuf = (torch.zeros_like(bn.weight), torch.zeros_like(bn.bias))
                st.g_own = torch.zeros(Cout, Cin, device=x.device, dtype=torch.float32)
            for t in st.gbuf + (st.g_own,):
                t.zero_()
            dg, db, gw = st.gbuf[0], st.gbuf[1], st.g_own
        # BatchNorm-backward statistics of dz = dy * act'(z), then dh = ca*dz + cb*h + cc
        q = nat.BnBwd()
        ws = engine.Workspace.get(x.device)
        q.partials, q.counter = ws.partials.data_ptr(), ws.counter.data_ptr()
        q.gamma = nat.ptr(bn.weight)
        q.mean, q.invstd = c_mean, c_invstd
        q.dgamma, q.dbeta = dg.data_ptr(), db.data_ptr()
        q.ca, q.cb, q.cc = b.ca.data_ptr(), b.cb.data_ptr(), b.cc.data_ptr()
        q.count = M
        q.use_batch_stats = 1 if b.batch_stats else 0
        r = nat.BnReduce()
        r.M, r.C, r.lddy, r.ldh = M, Cout, Cout, Cout
        r.dy, r.h, r.bn = dym.data_ptr(), hm.data_ptr(), C.pointer(q)
        r.z_scale, r.z_shift, r.z_act = c_scale, c_shift, act
        engine.launch(lib.yamb_bn_reduce_bwd, r, "bn_reduce", 4 * M * Cout)
        dh = torch.empty(M, Cout, device=x.device, dtype=torch.bfloat16)
        a = nat.BnBwdApply()
        a.M, a.C, a.lddy, a.ldh, a.lddh = M, Cout, Cout, Cout, Cout
        a.dy, a.h = dym.data_ptr(), hm.data_ptr()
        a.z_scale, a.z_shift, a.z_act = c_scale, c_shift, act
        a.ca, a.cb, a.cc = b.ca.data_ptr(), b.cb.data_ptr(), b.cc.data_ptr()
        a.dh = dh.data_ptr()
        engine.launch(lib.yamb_bn_bwd_apply_bwd, a, "bn_bwd_apply", 6 * M * Cout)
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
        g2 = _gemm(Cout, Cin, M, dh.data_ptr(), Cout, xm.data_ptr(), Cin, gw.data_ptr(), Cin,
                   a_mn_major=1, b_mn_major=1, epi=2)
        engine.launch(lib.yamb_pointwise_gemm, g2, "head_conv_wgrad", 2 * M * (Cin + Cout),
                      2 * M * Cin * Cout)
        if direct:
            return dx, None, None, None, None, None
        return dx, None, None, gw.view_as(conv.weight).clone(), dg.clone(), db.clone()


def pw_conv_bn_act(mod, x):
    """ConvBNReLU with a 1x1 convolution (reference models/mobilenet_base.py:181-203) on CUDA."""
    x = engine.to_nhwc_bf16(x)
    conv, bn, act = mod[0], mod[1], mod[2]
    return _PwConvBnActFn.apply(x, mod, engine.act_code_of(act), conv.weight, bn.weight, bn.bias)


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
        self.g_own = None
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
        ctx.lin, ctx.st = lin, st
        ctx.save_for_backward(x, wbf)
        return y

    @staticmethod
    def backward(ctx, dy):
        lib = nat.lib()
        x, wbf = ctx.saved_tensors
        lin, st = ctx.lin, ctx.st
        M, I = x.shape
        O = lin.out_features
        dy = dy.contiguous()
        if dy.dtype != torch.bfloat16:
            dy = dy.to(torch.bfloat16)
        direct = all(getattr(p, "_yamb_direct", False) and p.grad is not None
                     for p in (lin.weight, lin.bias))
        if direct:
            gw = lin.weight.grad
        else:
            if st.g_own is None:
                st.g_own = torch.zeros(O, I, device=x.device, dtype=torch.float32)
            st.g_own.zero_()
            gw = st.g_own
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
        if direct:
            gb_t = lin.bias.grad
        else:
            gb_t = torch.zeros(O, device=x.device, dtype=torch.float32)
        nat.check(lib.yamb_colsum_bf16(dy.data_ptr(), M, O, O, gb_t.data_ptr(), nat.stream_handle()))
        engine.LAUNCHES += 1
        if direct:
            return dx, None, None, None
        return dx, None, gw.clone(), gb_t


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
class _StemConvFn(torch.autograd.Function):
    """Raw output of the 3x3 / stride-2 / 3-channel first convolution (reference
    models/mobilenet_supernet.py:124-130) by the direct kernels of csrc/stem.cu; weight gradient
    in backward, no input gradient."""

    @staticmethod
    def forward(ctx, x, conv, weight):
        lib = nat.lib()
        N, _, H, W = x.shape
        Cout = conv.out_channels
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        y = torch.empty((N, Cout, Ho, Wo), device=x.device, dtype=torch.bfloat16,
                        memory_format=torch.channels_last)
        a = nat.StemConv()
        a.N, a.H, a.W, a.Cout = N, H, W, Cout
        a.x, a.w, a.y = x.data_ptr(), conv.weight.data_ptr(), y.data_ptr()
        engine.launch(lib.yamb_stem_conv_fwd, a, "stem_conv_fwd",
                      2 * N * (H * W * 3 + Ho * Wo * Cout), 2 * N * Ho * Wo * Cout * 27)
        ctx.conv = conv
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
        w = conv.weight
        direct = getattr(w, "_yamb_direct", False) and w.grad is not None
        gw = w.grad if direct else torch.zeros_like(w, dtype=torch.float32)
        a = nat.StemConv()
        a.N, a.H, a.W, a.Cout = N, H, W, Cout
        a.x, a.dh, a.dw = x.data_ptr(), dh.data_ptr(), gw.data_ptr()
        engine.launch(lib.yamb_stem_conv_wgrad, a, "stem_conv_wgrad",
                      2 * N * (H * W * 3 + dh.shape[2] * dh.shape[3] * Cout),
                      2 * N * dh.shape[2] * dh.shape[3] * Cout * 27)
        return None, None, (None if direct else gw)


def stem_supported(mod, x):
    conv, bn, act = mod[0], mod[1], mod[2]
    co = conv.out_channels
    return (x.is_cuda and conv.in_channels == 3 and conv.kernel_size == (3, 3)
            and conv.stride == (2, 2) and conv.padding == (1, 1) and conv.groups == 1
            and conv.dilation == (1, 1) and conv.bias is None and co in (8, 16, 32, 64)
            and bn.affine
            and type(act).__name__ in ("ReLU", "ReLU6", "Swish", "HSwish", "Identity"))


def stem_conv_bn_act(mod, x):
    """ConvBNReLU(3, C, stride=2) on CUDA: direct convolution kernel -> BatchNorm statistics ->
    BatchNorm apply + activation (engine.bn_act_apply)."""
    x = engine.to_nhwc_bf16(x)
    conv, bn, act = mod[0], mod[1], mod[2]
    h = _StemConvFn.apply(x, conv, conv.weight)
    return engine.bn_act_apply(bn, act, h)
