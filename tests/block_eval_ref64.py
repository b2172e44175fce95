"""Float64 reference of the one-launch eval block (csrc/block_eval.cuh) with rounding intervals.

The kernel's rounding points (header, "Rounding points"):
    a1 = bf16(act(bn1(acc32)))     acc32: the expand MMA over Cin in fp32
    a2 = bf16(act(bn2(sten32)))    sten32: the k x k stencil of a1 in fp32
    a2s = bf16(a2 * gate)          Squeeze-and-Excitation gate
    y = bf16(bn3(acc32) + x)       acc32: the project MMA over Chid (+ the cluster partials)
    pooled = fp32 mean of a2       pool pass

Every bf16 stage is carried as [lo, hi], the smallest and largest bf16 value the kernel may store.
Each bound is the fp64 value of the stage over the intervals of its inputs (per-term signs for the
sums; the minimum of Swish / h-swish when it lies inside), widened by a rigorous bound on the fp32
error ahead of the rounding, then rounded to fp32 outward and to bf16 to nearest (rounding is
monotone, so the stored value lies between the rounded ends).  The fp32 error bounds:
    * a length-n sum: n * 2^-23 * sum|terms| for the MMAs (one ulp per addition: the tensor
      cores' accumulation need not round to nearest), (n + 1) * 2^-24 * sum|terms| for the
      round-to-nearest fp32 chains of the stencil and the pool sums;
    * the BatchNorm fold scale = gamma * rsqrtf(var + eps), shift = beta - mean * scale, with
      rsqrtf at 2 ulp: |scale error| <= 2^-21 |scale|, |shift error| <= (2^-21 + 2^-23) |mean *
      scale| + 2^-23 |beta|; one rounding for each fmaf / add that follows;
    * Swish as __fdividef(z, 1 + __expf(-z)): relative (8 + 2|z|) 2^-23 (__expf: 2 + 1.173|z| ulp,
      __fdividef: 2 ulp); h-swish: three fp32 roundings.
Tensors are NCHW float64 on the device of the inputs."""
import torch
import torch.nn.functional as F

import ref64

U23 = 2.0 ** -23
U24 = 2.0 ** -24
ES = 2.0 ** -21          # relative error of the folded BatchNorm scale
SWISH_ZMIN = -1.2784645427610738   # argmin of z * sigmoid(z)


# ---- rounding ------------------------------------------------------------------------------------
def _f32_down(v):
    f = v.float()
    return torch.where(f.double() > v, torch.nextafter(f, torch.full_like(f, -float("inf"))), f)


def _f32_up(v):
    f = v.float()
    return torch.where(f.double() < v, torch.nextafter(f, torch.full_like(f, float("inf"))), f)


def bf16_interval(lo, hi):
    """[lo, hi] (fp64 reals) -> the bf16 values round-to-nearest of any fp32 inside can give."""
    return (_f32_down(lo).to(torch.bfloat16).double(), _f32_up(hi).to(torch.bfloat16).double())


# ---- BatchNorm fold ------------------------------------------------------------------------------
def bn_fold(bn):
    """(scale, shift, scale error, shift error) in fp64 of a dict gamma / beta (None: 1 / 0), mean,
    var, eps."""
    var, mean = bn["var"].double(), bn["mean"].double()
    g = bn["gamma"].double() if bn["gamma"] is not None else torch.ones_like(var)
    b = bn["beta"].double() if bn["beta"] is not None else torch.zeros_like(var)
    s = g / torch.sqrt(var + float(torch.tensor(bn["eps"], dtype=torch.float32)))
    t = b - mean * s
    return s, t, ES * s.abs(), (ES + U23) * (mean * s).abs() + U23 * b.abs()


def _c(v):
    return v.view(1, -1, 1, 1)


def affine_interval(lo, hi, s, t, es, et, extra=None):
    """fmaf(scale, v, shift) for v in [lo, hi] (the channel on dim 1), fp32 rounding included.
    extra: a further addend [e_lo, e_hi] (the residual), added in a second fp32 rounding."""
    s4, t4, es4, et4 = _c(s), _c(t), _c(es), _c(et)
    a, b = s4 * lo + t4, s4 * hi + t4
    zlo, zhi = torch.minimum(a, b), torch.maximum(a, b)
    m = torch.maximum(lo.abs(), hi.abs())
    err = es4 * m + et4 + U24 * ((s4.abs() + es4) * m + t4.abs() + et4)
    zlo, zhi = zlo - err, zhi + err
    if extra is not None:
        zlo, zhi = zlo + extra, zhi + extra
        r = U24 * torch.maximum(zlo.abs(), zhi.abs())
        zlo, zhi = zlo - r, zhi + r
    return zlo, zhi


# ---- activation ----------------------------------------------------------------------------------
def act_interval(lo, hi, act):
    """act over [lo, hi] widened by the error of the kernel's fp32 activation."""
    if act in (0, 1, 2):
        return ref64._clamp32(lo, act), ref64._clamp32(hi, act)   # clamps of the rounded value
    alo, ahi = ref64._act(lo, act), ref64._act(hi, act)
    top = torch.maximum(alo, ahi)
    zmin = SWISH_ZMIN if act == 3 else -1.5
    bot = torch.where((lo < zmin) & (hi > zmin), ref64._act(torch.full_like(lo, zmin), act),
                      torch.minimum(alo, ahi))
    m = torch.maximum(lo.abs(), hi.abs())
    amax = torch.maximum(bot.abs(), top.abs())
    if act == 3:
        err = amax * (8 + 2 * m) * U23
    else:
        err = U23 * (2 * amax + m * (m + 3) / 6)
    return bot - err, top + err


# ---- stages --------------------------------------------------------------------------------------
def expand(x, w1, bn1, act):
    """a1 interval [N, Chid, H, W] of x [N, Cin, H, W] (bf16 values) and W1 [Chid, Cin]."""
    x, w1 = x.double(), w1.double()
    h = torch.einsum("nchw,dc->ndhw", x, w1)
    err = x.shape[1] * U23 * torch.einsum("nchw,dc->ndhw", x.abs(), w1.abs())
    s, t, es, et = bn_fold(bn1)
    zlo, zhi = affine_interval(h - err, h + err, s, t, es, et)
    return bf16_interval(*act_interval(zlo, zhi, act))


def stencil(a_lo, a_hi, wdw, k, stride, bn2, act):
    """a2 interval [N, Chid, Ho, Wo] of the a1 interval (zero outside the image) and the depthwise
    weights [Chid, k*k] (fp32)."""
    C = a_lo.shape[1]
    w = wdw.double().view(C, 1, k, k)
    wp, wm = w.clamp(min=0), w.clamp(max=0)
    conv = lambda v, ww: F.conv2d(v, ww, stride=stride, padding=(k - 1) // 2, groups=C)
    lo = conv(a_lo, wp) + conv(a_hi, wm)
    hi = conv(a_hi, wp) + conv(a_lo, wm)
    err = (k * k + 1) * U24 * conv(torch.maximum(a_lo.abs(), a_hi.abs()), w.abs())
    s, t, es, et = bn_fold(bn2)
    zlo, zhi = affine_interval(lo - err, hi + err, s, t, es, et)
    return bf16_interval(*act_interval(zlo, zhi, act))


def gated(a_lo, a_hi, gate):
    """a2s = bf16(fp32(a2 * gate[n][c]))."""
    g = gate.double()[:, :, None, None]
    p, q = a_lo * g, a_hi * g
    return bf16_interval(torch.minimum(p, q), torch.maximum(p, q))


def project(a_lo, a_hi, w3, bn3, x=None, extra_adds=0):
    """y interval [N, Cout, Ho, Wo]: the project over Chid (extra_adds: the cluster's partial
    sums), bn3 and the residual x (bf16 values) when given."""
    w = w3.double()
    wp, wm = w.clamp(min=0), w.clamp(max=0)
    mm = lambda v, ww: torch.einsum("nchw,dc->ndhw", v, ww)
    lo = mm(a_lo, wp) + mm(a_hi, wm)
    hi = mm(a_hi, wp) + mm(a_lo, wm)
    err = (w.shape[1] + extra_adds) * U23 * mm(torch.maximum(a_lo.abs(), a_hi.abs()), w.abs())
    s, t, es, et = bn_fold(bn3)
    zlo, zhi = affine_interval(lo - err, hi + err, s, t, es, et,
                               None if x is None else x.double())
    return bf16_interval(zlo, zhi)


def pooled(a_lo, a_hi, nslab):
    """pooled interval [N, Chid] (fp32 values, not rounded further): the mean of a2 over the
    output pixels, run / tile / slab sums and the multiply by fp32(1 / (Ho * Wo))."""
    hw = a_lo.shape[2] * a_lo.shape[3]
    lo, hi = a_lo.sum((2, 3)) / hw, a_hi.sum((2, 3)) / hw
    m = torch.maximum(a_lo.abs(), a_hi.abs()).sum((2, 3)) / hw
    err = (hw + nslab + 4) * U24 * m
    return lo - err, hi + err


def count_values(lo, hi):
    """bf16 values in [lo, hi] (both bf16 values)."""
    def key(v):
        i = v.to(torch.bfloat16).view(torch.int16).int()
        return torch.where(i < 0, -(i & 0x7FFF), i)
    return key(hi) - key(lo) + 1
