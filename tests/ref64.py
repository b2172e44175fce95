"""Float64 references and element-by-element checkers shared by the GPU kernel tests
(test_bn_elementwise_gpu.py, test_gemm_fp64_gpu.py, test_depthwise_gpu.py).

Staged values.  An fmaf(a, b, c) of an fp32 and a bf16 operand is reproduced by forming the sum in
fp64 (the product is exact there) and rounding once to fp32.  Swish and h-swish run on __expf /
__fdividef: where the exact value lies within BAND (relative) of a bf16 rounding boundary the
stored value may sit one bf16 ulp away.

Long sums: with r the fp64 reference and Q = sqrt(sum term^2), |got - r| <= 2^-10 |r| + 2^-8 Q
(_long_bound).  A missing tile of rows changes such a sum by a multiple of Q.

Derived BatchNorm values (mean, invstd, scale, shift, running statistics, ca / cb / cc) carry the
bound propagated through the fp64 derivation, plus the fp32 rounding of the stored value; the
running statistics are checked against torch.nn.BatchNorm2d itself."""
import torch

SENTINEL = -1536.0       # a bf16 value no output of these tests takes
POISON = 4096.0          # fills the input row after M: a kernel that reads it is far off
BAND = 2.0 ** -16
DEV = "cuda"


# ---- activations ---------------------------------------------------------------------------------
def _act(z, act):
    """act(z) in z's dtype (plain torch expressions of the five activation codes)."""
    if act == 1:
        return torch.relu(z)
    if act == 2:
        return torch.clamp(z, 0, 6)
    if act == 3:
        return z * torch.sigmoid(z)
    if act == 4:
        return z * torch.clamp(z + 3, 0, 6) / 6
    return z


def _act_grad(z, act):
    """act'(z) in fp32 (plain torch expressions; 0 at the ReLU / ReLU6 edges)."""
    if act == 1:
        return (z > 0).float()
    if act == 2:
        return ((z > 0) & (z < 6)).float()
    if act == 3:
        s = torch.sigmoid(z)
        return s * (1 + z * (1 - s))
    if act == 4:
        return torch.where(z <= -3, torch.zeros_like(z),
                           torch.where(z >= 3, torch.ones_like(z), (2 * z + 3) / 6))
    return torch.ones_like(z)


def _act_mod(act):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    return {0: torch.nn.Identity(), 1: torch.nn.ReLU(), 2: torch.nn.ReLU6(), 3: mb.Swish(),
            4: mb.HSwish()}[act]


def _act64(z, act):
    with torch.no_grad():
        return _act_mod(act)(z.double())


def _dact64(z, act):
    """d act / dz in fp64 by autograd through the reference's activation module."""
    z = z.double().detach().requires_grad_(True)
    with torch.enable_grad():
        y = _act_mod(act)(z)
        (g,) = torch.autograd.grad(y, z, torch.ones_like(y))
    return g


def _clamp32(z, act):
    if act == 1:
        return torch.clamp(z, min=0.0)
    if act == 2:
        return torch.clamp(z, 0.0, 6.0)
    return z


def _act_err(z, act, g):
    """Bound on |act'(z) computed with the kernel's fp32 intrinsics - exact|."""
    if act == 3:
        return 2.0 ** -18 * (1 + z.abs())
    if act == 4:
        return 2.0 ** -21 * g.abs()
    return torch.zeros_like(z)


# ---- data ----------------------------------------------------------------------------------------
def _f32(t):
    return t.double().float()


def _bf(shape, scale=1.0, shift=0.0, gen=None):
    return (torch.randn(shape, device=DEV, generator=gen) * scale + shift).to(torch.bfloat16)


def _with_poison(t):
    """[M, ld] -> [M + 1, ld] with a poison row after M."""
    return torch.cat([t, torch.full((1, t.shape[1]), POISON, device=DEV, dtype=t.dtype)])


def _guarded(n, fill=0.0, dtype=torch.float32):
    """n values followed by 8 guard values that must keep SENTINEL."""
    t = torch.full((n + 8,), SENTINEL, device=DEV, dtype=dtype)
    t[:n] = fill
    return t


# ---- checks --------------------------------------------------------------------------------------
def _check_guard(t, n, what):
    assert bool((t[n:] == SENTINEL).all()), "%s: written past its %d values" % (what, n)


def _check_zero(partials, counter):
    assert int(counter.item()) == 0, "counter not returned to 0"
    assert float(partials.abs().max()) == 0.0, "BatchNorm accumulator not returned to 0"


def _same(a, b, what):
    assert torch.equal(a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8)), \
        "%s: bits differ between two identical calls" % what


def _check_frame(buf, M, c0, C, what):
    """Rows [0, M) outside the channel slice and the row after M keep SENTINEL."""
    ok = bool((buf[:M, :c0] == SENTINEL).all()) and bool((buf[:M, c0 + C:] == SENTINEL).all())
    assert ok, "%s: wrote channels outside [%d, %d)" % (what, c0, c0 + C)
    assert bool((buf[M] == SENTINEL).all()), "%s: wrote the row after M" % what


def _fail(what, idx, loc, detail):
    msg = "%s: %s at %s" % (what, detail, idx)
    if loc is not None:
        msg += " " + loc(*idx)
    raise AssertionError(msg)


def _worst(err, bound, what, loc=None):
    """Largest err / bound; on failure name the element and where the grid walk produced it."""
    ratio = err / (bound + 1e-300)
    i = int(ratio.argmax())
    r = float(ratio.flatten()[i])
    if not r <= 1.0:
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), ratio.shape))
        _fail(what, idx, loc, "err/bound %.3g (got-ref %.4g, bound %.4g)"
              % (r, float(err.flatten()[i]), float(bound.flatten()[i])))
    return r


def _equal(got, want, what, loc=None):
    """Equal values (bf16 / fp32; +0 == -0)."""
    bad = got.double() != want.double()
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), bad.shape))
        _fail(what, idx, loc, "got %r want %r (%d elements differ)"
              % (float(got.flatten()[i]), float(want.flatten()[i]), int(bad.sum())))


def _outside(got, y64, delta):
    """Mask of the elements of got (bf16) outside the bf16 values of y64 -+ delta."""
    lo = (y64 - delta).float().to(torch.bfloat16).double()
    hi = (y64 + delta).float().to(torch.bfloat16).double()
    g = got.double()
    return (g < lo) | (g > hi) | ~torch.isfinite(g), lo, hi


def _between(got, y64, delta, what, loc=None):
    """got (bf16) must lie between the bf16 values of y64 -+ delta."""
    bad, lo, hi = _outside(got, y64, delta)
    if bool(bad.any()):
        g = got.double()
        i = int(bad.flatten().nonzero()[0])
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), bad.shape))
        _fail(what, idx, loc, "got %r outside [%r, %r] (exact %r; %d elements)"
              % (float(g.flatten()[i]), float(lo.flatten()[i]), float(hi.flatten()[i]),
                 float(y64.flatten()[i]), int(bad.sum())))


def _long_bound(r, q):
    return 2.0 ** -10 * r.abs() + 2.0 ** -8 * q


def _staged_band(a):
    lo = (a * (1 - BAND)).float().to(torch.bfloat16).double()
    hi = (a * (1 + BAND)).float().to(torch.bfloat16).double()
    return (hi - lo).abs()


# ---- BatchNorm structs ---------------------------------------------------------------------------
def _nat():
    from yet_another_mobilenet_series_b200 import native as nat
    return nat


class _Acc:
    """Statistics accumulator (2*C doubles + guard) and arrival counter."""

    def __init__(self, C):
        self.C = C
        self.partials = torch.zeros(2 * C + 64, device=DEV, dtype=torch.float64)
        self.counter = torch.zeros(1, device=DEV, dtype=torch.int32)

    def check(self):
        torch.cuda.synchronize()
        _check_zero(self.partials, self.counter)


def _bn_bwd(acc, C, count, gamma, mean, invstd, out, use_batch_stats=1):
    nat = _nat()
    b = nat.BnBwd()
    b.partials, b.counter = acc.partials.data_ptr(), acc.counter.data_ptr()
    b.gamma = None if gamma is None else gamma.data_ptr()
    b.mean, b.invstd = mean.data_ptr(), invstd.data_ptr()
    b.dgamma = None if out["dg"] is None else out["dg"].data_ptr()
    b.dbeta = None if out["db"] is None else out["db"].data_ptr()
    b.ca, b.cb, b.cc = out["ca"].data_ptr(), out["cb"].data_ptr(), out["cc"].data_ptr()
    b.count = count
    b.use_batch_stats = use_batch_stats
    return b


def _bwd_outputs(C, dg0, db0):
    out = {k: _guarded(C) for k in ("ca", "cb", "cc", "dg", "db")}
    out["dg"][:C] = dg0
    out["db"][:C] = db0
    return out


def _check_fwd_finalize(o, h64, gamma, beta, rm0, rv0, nbt0, eps, mom, b_s, b_q, what, loc):
    """mean / invstd / scale / shift and the running statistics of bn_fwd_finalize against the
    fp64 derivation from the column sums (bounds b_s, b_q) and against nn.BatchNorm2d's update of
    the running statistics.  o: the guarded outputs scale / shift / mean / invstd / rm / rv / nbt
    (rm / rv None: no running statistics).  Returns (mean_ref, var_ref, inv_ref)."""
    M, Cc = h64.shape
    ref = torch.nn.BatchNorm2d(Cc, eps=eps, momentum=mom, affine=gamma is not None).to(DEV).double()
    with torch.no_grad():
        ref.running_mean.copy_(rm0)
        ref.running_var.copy_(rv0)
        ref.num_batches_tracked.fill_(nbt0)
        ref.train()
        ref(h64.view(M, Cc, 1, 1))
    if o.get("nbt") is not None:
        assert int(o["nbt"]) == int(ref.num_batches_tracked) == nbt0 + 1, what + " num_batches_tracked"
    s_ref, q_ref = h64.sum(0), (h64 * h64).sum(0)
    mean_ref = s_ref / M
    var_ref = h64.var(0, unbiased=False)
    e_mean = b_s / M
    e_var = b_q / M + 2 * mean_ref.abs() * e_mean + e_mean ** 2
    inv_ref = (var_ref + eps).rsqrt()
    lo = (var_ref + eps - e_var).clamp_min(1e-300)
    e_inv = 0.5 * e_var * lo ** -1.5 + 2.0 ** -23 * inv_ref
    inv_got = None
    if o.get("mean") is not None:
        mean_got, inv_got = o["mean"][:Cc], o["invstd"][:Cc]
        _worst((mean_got.double() - mean_ref).abs(), e_mean + 2.0 ** -23 * mean_ref.abs(),
               what + " mean", loc)
        _worst((inv_got.double() - inv_ref).abs(), e_inv, what + " invstd", loc)
    g1 = gamma if gamma is not None else torch.ones(Cc, device=DEV)
    b1 = beta if beta is not None else torch.zeros(Cc, device=DEV)
    if inv_got is not None:
        scl = g1 * inv_got
        _equal(o["scale"][:Cc], scl, what + " scale = gamma * invstd", loc)
        _worst((o["shift"][:Cc].double() - (b1.double() - mean_got.double() * scl.double())).abs(),
               2.0 ** -22 * (b1.double().abs() + (mean_got * scl).double().abs()) + 1e-30,
               what + " shift", loc)
    else:
        scl_ref = g1.double() * inv_ref
        _worst((o["scale"][:Cc].double() - scl_ref).abs(),
               g1.double().abs() * e_inv + 2.0 ** -23 * scl_ref.abs(), what + " scale", loc)
        sh_ref = b1.double() - mean_ref * scl_ref
        _worst((o["shift"][:Cc].double() - sh_ref).abs(),
               (mean_ref.abs() * g1.double().abs() * e_inv + e_mean * scl_ref.abs()) * 1.01 +
               2.0 ** -21 * (b1.double().abs() + (mean_ref * scl_ref).abs()) + 1e-30,
               what + " shift", loc)
    if o.get("rm") is not None:
        fac = mom if mom is not None else 1.0 / (nbt0 + 1)
        unb = M / (M - 1)
        rnd = lambda a, b: 2.0 ** -22 * ((1 - fac) * a.abs() + fac * b.abs())
        _worst((o["rm"][:Cc].double() - ref.running_mean).abs(),
               fac * e_mean + rnd(rm0.double(), mean_ref), what + " running_mean", loc)
        _worst((o["rv"][:Cc].double() - ref.running_var).abs(),
               fac * e_var * unb + rnd(rv0.double(), var_ref * unb), what + " running_var", loc)
    return mean_ref, var_ref, inv_ref


def _check_bwd_finalize(out, C, M, gamma, mean1, invstd1, s_ref, q_ref, b_s, b_q, dg0, db0, what,
                        loc):
    """dgamma / dbeta (+=), ca / cb / cc of bn_bwd_finalize against the fp64 derivation."""
    for k in ("ca", "cb", "cc", "dg", "db"):
        if out[k] is not None:
            _check_guard(out[k], C, what + " " + k)
    g1 = torch.ones(C, device=DEV) if gamma is None else gamma
    acc = lambda p, r: 2.0 ** -23 * (p.double().abs() + r.abs())
    worst = {}
    if out["db"] is not None:
        worst["dbeta"] = _worst((out["db"][:C].double() - db0.double() - s_ref).abs(),
                                b_s + acc(db0, s_ref), what + " dbeta", loc)
    if out["dg"] is not None:
        worst["dgamma"] = _worst((out["dg"][:C].double() - dg0.double() - q_ref).abs(),
                                 b_q + acc(dg0, q_ref), what + " dgamma", loc)
    scl = g1 * invstd1
    _equal(out["ca"][:C], scl, what + " ca = gamma * invstd", loc)
    sr = scl.double() * invstd1.double()
    m1, m2 = s_ref / M, q_ref / M
    cb_ref = -sr * m2
    cc_ref = scl.double() * (mean1.double() * invstd1.double() * m2 - m1)
    mr = (mean1 * invstd1).double().abs()
    worst["cb"] = _worst((out["cb"][:C].double() - cb_ref).abs(),
                         sr.abs() * b_q / M + 2.0 ** -21 * cb_ref.abs() + 1e-30, what + " cb", loc)
    worst["cc"] = _worst((out["cc"][:C].double() - cc_ref).abs(),
                         scl.double().abs() * (mr * b_q / M + b_s / M) +
                         2.0 ** -21 * scl.double().abs() * (mr * m2.abs() + m1.abs()) + 1e-30,
                         what + " cc", loc)
    return worst


def _eval_mode_coeffs(run, out1, C, gamma, invstd1, what):
    """use_batch_stats = 0 (eval-mode BatchNorm): cb = cc = 0, ca = gamma * invstd, the same
    dgamma / dbeta."""
    out0 = run(0)
    g1 = torch.ones(C, device=DEV) if gamma is None else gamma
    _equal(out0["ca"][:C], g1 * invstd1, what + " eval-mode ca")
    assert float(out0["cb"][:C].abs().max()) == 0.0 and float(out0["cc"][:C].abs().max()) == 0.0, \
        what + ": eval-mode cb / cc not zero"
    for k in ("dg", "db"):
        if out1[k] is not None:
            _same(out0[k], out1[k], what + " eval-mode " + k)
    return out0
