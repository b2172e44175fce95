"""Float64 references and element checkers of the Squeeze-and-Excitation fully connected layers
(csrc/se_fc.cu), the non-local products (csrc/nonlocal.cu) and the non-local InstanceNorm
(csrc/instance_norm.cu), shared by test_se_nl_fp64_gpu.py (kernel outputs on the GPU) and
test_se_nl_plan_cpu.py (the same checkers on CPU data with planted faults).  Every function here
works on tensors of any device.  u = 2^-24.

fp32 FMA chains.  A sum formed by n roundings (fmaf steps, slab adds, the bias or scale step) of
terms whose absolute values add to A is within gam(n) A of the exact sum, gam(n) = n u / (1 - n u)
(Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., §3.1).  The chain length is the
one the launch plan implies: k_per_slab + slabs + 1 for the split-K SE products, K for the
single-slab ones, rows per chunk + chunks + 1 for the gram, K + 1 for the row x matrix product,
pixels per lane + 1 for the InstanceNorm sums.  A missing 16-wide K chunk, row chunk or sample
slab moves an element by the sum of its terms, orders of magnitude more than gam(n) A at these
lengths (test_se_nl_plan_cpu.py plants each).

Staged values.  A stage that reads an earlier stage's stored output is checked from that output
(gate from the kernel's v, du from its dt and u, dpool and the weight gradients from its du / dt,
InstanceNorm y / dh from its mean / invstd); each stored output has its own check."""
import torch

from ref64 import (_act64, _act_err, _between, _clamp32, _dact64, _equal, _fail,
                   _outside, _worst)

U = 2.0 ** -24
TINY = 2.0 ** -126            # flushed intrinsic results (ex2.approx.ftz, __fdividef's range)


def gam(n):
    return n * U / (1 - n * U)


def span_share(y64, delta):
    """Share of the elements whose bf16 interval [bf16(y64 - delta), bf16(y64 + delta)] holds
    more than two bf16 values (where the check is weak)."""
    _, lo, hi = _outside(y64.new_zeros(()).expand_as(y64), y64, delta)

    def key(t):
        b = t.float().to(torch.bfloat16).view(torch.int16).int()
        return torch.where(b >= 0, b, -(b & 0x7fff))
    return float(((key(hi) - key(lo) + 1) > 2).double().mean()) if y64.numel() else 0.0


def bf16_ratio(got, y64, delta):
    """Largest |got - y64| / (delta + 2^-8 (|y64| + delta)): the fp32 error bound plus the one bf16
    rounding, half a bf16 ulp (<= 1 for every value of the bf16 interval _between accepts)."""
    g = got.double()
    r = (g - y64).abs() / (delta + 2.0 ** -8 * (y64.abs() + delta) + 1e-300)
    return float(r.max()) if r.numel() else 0.0


def _d(t):
    return t.double()


# ---- Squeeze-and-Excitation ----------------------------------------------------------------------
def se_u_check(pooled, w_r, b_r, u, plan, what, loc=None):
    """u = W_r s + b_r: split-K chain of k_per_slab fmas, slabs added in order, then b_r."""
    r = _d(pooled) @ _d(w_r).t() + _d(b_r)
    A = _d(pooled).abs() @ _d(w_r).abs().t() + _d(b_r).abs()
    n = plan.split.k_per_slab + plan.split.nslab + 1
    return _worst((_d(u) - r).abs(), 1.01 * gam(n) * A, what, loc)


def se_v_check(u, v, act, what, loc=None):
    """v = act(u) on the kernel's u: exact for none / ReLU / ReLU6; Swish is __fdividef(z,
    1 + __expf(-z)) ((2 + 1.173 |z|) ulp for the exp, u for the add, 2 ulp for the division, 0
    once 1 + exp(-z) passes 2^126), h-swish three fp32 roundings and fp32(1/6)."""
    if act in (0, 1, 2):
        _equal(v, _clamp32(u.float(), act), what, loc)
        return 0.0
    z = _d(u)
    a64 = _act64(z, act)
    if act == 3:
        rel = ((2 + 1.173 * z.abs()) * 2.0 ** -23 + 3 * 2.0 ** -23) * 1.01
        bound = a64.abs() * rel + torch.where(z < -80, a64.abs(), torch.zeros_like(z)) + TINY
    else:
        bound = 2.0 ** -21 * a64.abs() + TINY
    return _worst((_d(v) - a64).abs(), bound, what, loc)


def se_gate_check(v, w_e, b_e, gate, what, loc=None):
    """gate = 1 / (1 + __expf(-t)), t = W_e v + b_e (R fmas + the bias), IEEE division."""
    t = _d(v) @ _d(w_e).t() + _d(b_e)
    A = _d(v).abs() @ _d(w_e).abs().t() + _d(b_e).abs()
    R = v.shape[1]
    et = gam(R + 1) * A
    s = torch.sigmoid(t)
    bound = s * (1 - s) * (et + (2 + 1.173 * (t.abs() + et)) * 2.0 ** -23) * 1.02 + \
        2.02 * U * s + TINY
    return _worst((_d(gate) - s).abs(), bound, what, loc)


def se_dt_check(dgate, gate, dt, what, loc=None):
    """dt = (dgate * g) * (1 - g): three fp32 roundings, no add to contract: bit for bit."""
    g = gate.float()
    _equal(dt, (dgate.float() * g) * (1 - g), what, loc)


def colsum_check(got, g0, x, rows, slabs, what, loc=None):
    """got = g0 + sum over samples of x, as slabs of `rows` samples each summed in sample order
    (fp32), the slabs added in slab order, then added onto g0."""
    r = _d(x).sum(0)
    A = _d(x).abs().sum(0)
    e = gam(min(rows, x.shape[0]) + slabs) * A
    bound = 1.01 * (e + U * (_d(g0).abs() + r.abs() + e))
    return _worst((_d(got) - _d(g0) - r).abs(), bound, what, loc)


def se_du_check(dt, w_e, u, act, du, plan, what, loc=None):
    """du = (W_e^T dt) * act'(u): the split-K chain of u's plan, one product with act'(u_saved);
    act' is exact for none / ReLU / ReLU6 and within _act_err for Swish / h-swish."""
    a = _d(dt) @ _d(w_e)
    A = _d(dt).abs() @ _d(w_e).abs()
    ea = gam(plan.split.k_per_slab + plan.split.nslab) * A
    g = _dact64(_d(u), act)
    eg = _act_err(_d(u), act, g)
    bound = 1.01 * (ea * (g.abs() + eg) + a.abs() * eg + U * (a.abs() + ea) * (g.abs() + eg))
    return _worst((_d(du) - a * g).abs(), bound, what, loc)


def se_dpool_check(du, w_r, inv_hw, dpool, what, loc=None):
    """dpool = inv_hw * (du W_r): R fmas, then the scale."""
    al = float(torch.tensor(inv_hw, dtype=torch.float32))
    r = al * (_d(du) @ _d(w_r))
    A = al * (_d(du).abs() @ _d(w_r).abs())
    return _worst((_d(dpool) - r).abs(), 1.01 * (gam(du.shape[1]) * A + U * r.abs()), what, loc)


def gemm_acc_check(got, g0, a, b, what, loc=None):
    """got = g0 + a^T b: one chain of a.shape[0] fmas, then the add onto g0."""
    r = _d(a).t() @ _d(b)
    A = _d(a).abs().t() @ _d(b).abs()
    e = gam(a.shape[0]) * A
    bound = 1.01 * (e + U * (_d(g0).abs() + r.abs() + e))
    return _worst((_d(got) - _d(g0) - r).abs(), bound, what, loc)


# ---- non-local products --------------------------------------------------------------------------
def rows_of(X, N, H, W, sub, width):
    """[N, rows, width] fp64 of the row set (pixels (::sub, ::sub) of each sample)."""
    return _d(X[:N * H * W, :width]).view(N, H, W, width)[:, ::sub, ::sub].reshape(N, -1, width)


def row_mask(N, H, W, sub, device):
    """[N*H*W] bool: the pixel is in the row set."""
    m = torch.zeros(N, H, W, dtype=torch.bool, device=device)
    m[:, ::sub, ::sub] = True
    return m.view(-1)


def gram_check(G, X, Y, N, H, W, sub, I, J, alpha, plan, what, loc=None):
    """G = alpha sum over the row set of X[:, :I]^T Y[:, :J] (bf16 products are exact in fp32):
    chains of rows-per-chunk fmas, the alpha step, chunks added in order."""
    xs, ys = rows_of(X, N, H, W, sub, I), rows_of(Y, N, H, W, sub, J)
    al = float(torch.tensor(alpha, dtype=torch.float32))
    r = al * (xs.transpose(1, 2) @ ys)
    A = abs(al) * (xs.abs().transpose(1, 2) @ ys.abs())
    return _worst((_d(G).view(N, I, J) - r).abs(), 1.01 * gam(plan.R + plan.chunks + 1) * A,
                  what, loc)


def rowmat_value(X, M3, N, H, W, sub, Kd, alpha):
    """(alpha X_rows M, |alpha| |X_rows| |M|), [N, rows, O], M3: [N, K, O] fp64."""
    xs = rows_of(X, N, H, W, sub, Kd)
    al = float(torch.tensor(alpha, dtype=torch.float32))
    return al * (xs @ M3), abs(al) * (xs.abs() @ M3.abs())


def rowmat_delta(r, A, b, Kd):
    """fp32 error before the bf16 rounding of out = b + alpha sum_k x_k m_k: K fmas, the alpha
    step, the add of the bf16 addend b."""
    return 1.02 * (gam(Kd) * A + U * r.abs() + U * (r + b).abs())


def rowmat_check(out, out0, X, M3, N, H, W, sub, Kd, O, alpha, base, accumulate, o_copy, what,
                 loc=None):
    """out [M + 1, ldo] after the call, out0 before it.  Rows of the row set, columns < O: within
    the bf16 interval of (base | out0 | 0) + alpha X M; columns [O, o_copy) with base: base's bits;
    every other element keeps its bits (SENTINEL frame, rows outside the row set)."""
    M = N * H * W
    r, A = rowmat_value(X, M3, N, H, W, sub, Kd, alpha)
    rows = row_mask(N, H, W, sub, out.device)
    idx = rows.nonzero().view(-1)
    if base is not None:
        b = _d(base[idx, :O]).view_as(r)
    elif accumulate:
        b = _d(out0[idx, :O]).view_as(r)
    else:
        b = torch.zeros_like(r)
    y64 = r + b
    delta = rowmat_delta(r, A, b, Kd)
    _between(out[idx, :O].view_as(r), y64, delta, what, loc)
    written = torch.zeros_like(out, dtype=torch.bool)
    written[idx, :O] = True
    if base is not None and o_copy > O:
        written[idx, O:o_copy] = True
        _equal(out[idx, O:o_copy], base[idx, O:o_copy], what + " pass-through columns")
    keep = ~written
    bad = keep & (out.view(torch.int16) != out0.view(torch.int16))
    if bool(bad.any()):
        i = bad.nonzero()[0].tolist()
        _fail(what, tuple(i), None, "wrote outside its rows / columns (M %d, O %d, o_copy %d)"
              % (M, O, o_copy))
    return y64, delta


# ---- InstanceNorm --------------------------------------------------------------------------------
def in_chain(HW, C, lanes, device):
    """[C] per-lane chain length + 1 (the h - K or h - mu rounding) of each channel's chunk."""
    ch = []
    for ln in lanes:
        ch += [-(-HW // ln.PX) + 1] * (8 * ln.CG)
    return torch.tensor(ch[:C], dtype=torch.float64, device=device)


def in_stats_check(h, N, HW, C, eps, mean, invstd, lanes, what, loc=None):
    """mean / invstd [N, C] against fp64: per-lane fp32 chains of d = h - h[first pixel] and d^2,
    lanes merged in double, var = E[d^2] - E[d]^2.  Returns (mean64, var64, e_mean, e_var)."""
    hv = _d(h[:N * HW, :C]).view(N, HW, C)
    d = hv - hv[:, :1]
    n = in_chain(HW, C, lanes, h.device)
    g = n * U / (1 - n * U) + 2.0 ** -50
    md = d.mean(1)
    e_md = g * d.abs().sum(1) / HW
    mean64 = hv.mean(1)
    var64 = hv.var(1, unbiased=False)
    e_var = g * (d * d).sum(1) / HW + 2 * md.abs() * e_md + e_md ** 2
    e_mean = e_md + U * mean64.abs() * 1.01
    ep = float(torch.tensor(eps, dtype=torch.float32))
    inv64 = (var64 + ep).rsqrt()
    lo = (var64 + ep - e_var).clamp_min(1e-300)
    e_inv = 1.01 * (0.5 * e_var * lo ** -1.5 + U * inv64)
    r = max(_worst((_d(mean) - mean64).abs(), e_mean, what + " mean", loc),
            _worst((_d(invstd) - inv64).abs(), e_inv, what + " invstd", loc))
    return mean64, var64, e_mean, e_var, r


def in_y_check(h, N, HW, C, gamma, beta, mean, invstd, res, res2, y, what, loc=None):
    """y = fmaf(sc, h, b - mean sc) (+ res) (+ res2), sc = fp32(gamma invstd), from the kernel's
    mean / invstd: a few fp32 roundings before the bf16 one."""
    M = N * HW
    inv = invstd.float().view(N, 1, C)
    g = gamma.float() if gamma is not None else torch.ones(C, device=h.device)
    b = _d(beta) if beta is not None else torch.zeros(C, dtype=torch.float64, device=h.device)
    sc = _d(g * inv)
    ms = _d(mean).view(N, 1, C) * sc
    sh = b - ms
    hv = _d(h[:M, :C]).view(N, HW, C)
    y64 = sc * hv + sh
    mag = (sc * hv).abs() + sh.abs()
    for t in (res, res2):
        if t is not None:
            rv = _d(t[:M, :C]).view(N, HW, C)
            y64 = y64 + rv
            mag = mag + rv.abs()
    delta = 1.01 * U * (b.abs() + 2 * ms.abs() + 3 * mag)
    _between(y[:M, :C].view(N, HW, C), y64, delta, what + " y", loc)
    return y64, delta


def in_running_check(h, N, HW, C, eps, mom, affine, rm0, rv0, rm, rv, e_mean, e_var, what):
    """Running statistics against torch.nn.InstanceNorm2d(track_running_stats=True) in fp64,
    within the propagated per-sample bounds and the fp32 update."""
    ref = torch.nn.InstanceNorm2d(C, eps=eps, momentum=mom, affine=affine,
                                  track_running_stats=True).to(h.device).double()
    x = _d(h[:N * HW, :C]).view(N, HW, C).permute(0, 2, 1).reshape(N, C, HW, 1)
    with torch.no_grad():
        ref.running_mean.copy_(rm0)
        ref.running_var.copy_(rv0)
        ref.train()
        ref(x)
    hv = _d(h[:N * HW, :C]).view(N, HW, C)
    unb = HW / (HW - 1)
    am, av = hv.mean(1).mean(0), (hv.var(1, unbiased=False) * unb).mean(0)
    rnd = lambda a, b: 2.0 ** -21 * ((1 - mom) * _d(a).abs() + mom * b.abs())   # noqa: E731
    return max(_worst((_d(rm) - ref.running_mean).abs(), mom * e_mean.mean(0) + rnd(rm0, am),
                      what + " running_mean"),
               _worst((_d(rv) - ref.running_var).abs(),
                      mom * (e_var * unb + U * hv.var(1) * 1.01).mean(0) + rnd(rv0, av),
                      what + " running_var"))


def in_bwd_check(dy, h, N, HW, C, gamma, mean, invstd, dh, lanes, what, loc=None):
    """dh = a (dy - m1 - xhat m2), a = fp32(gamma invstd), m1 = sum(dy) / HW, m2 = sum(dy (h -
    mu)) invstd / HW from the kernel's mean / invstd.  Returns (S, Q, e_S, e_Q) [N, C]: the
    per-sample sums of dy and dy (h - mu) and their bounds."""
    M = N * HW
    mu, rs = _d(mean).view(N, 1, C), _d(invstd).view(N, 1, C)
    hv = _d(h[:M, :C]).view(N, HW, C)
    dv = _d(dy[:M, :C]).view(N, HW, C)
    hm = hv - mu
    n = in_chain(HW, C, lanes, h.device)
    S, Q = dv.sum(1), (dv * hm).sum(1)
    e_S = (n * U / (1 - n * U) + 2.0 ** -50) * dv.abs().sum(1)
    e_Q = ((n + 1) * U / (1 - (n + 1) * U) + 2.0 ** -50) * (dv * hm).abs().sum(1)
    rs2 = rs.view(N, C)
    m1, m2 = (S / HW).view(N, 1, C), (Q * rs2 / HW).view(N, 1, C)
    e_m1 = (e_S / HW).view(N, 1, C) + 1.01 * U * m1.abs()
    e_m2 = (rs2.abs() * e_Q / HW).view(N, 1, C) + 1.01 * U * m2.abs()
    xh = hm * rs
    inner = dv - m1 - xh * m2
    e_in = 1.01 * (e_m1 + xh.abs() * e_m2 + 2.01 * U * xh.abs() * (m2.abs() + e_m2)) + \
        1.01 * U * (dv.abs() + m1.abs() + 2 * (xh * m2).abs() + inner.abs())
    g = gamma.float() if gamma is not None else torch.ones(C, device=h.device)
    a = _d(g * invstd.float().view(N, 1, C))
    dh64 = a * inner
    delta = 1.02 * (a.abs() * e_in + U * dh64.abs())
    _between(dh[:M, :C].view(N, HW, C), dh64, delta, what + " dh", loc)
    return S, Q * rs2, e_S, rs2.abs() * e_Q, dh64, delta


def in_param_check(got, g0, per_sample, e_per_sample, what):
    """dgamma / dbeta += the per-sample sums (stored as fp32, added in double in sample order)."""
    s = per_sample.sum(0)
    bound = 1.01 * ((e_per_sample + U * per_sample.abs()).sum(0) + U * s.abs() +
                    U * (_d(g0).abs() + (_d(g0) + s).abs()))
    return _worst((_d(got) - _d(g0) - s).abs(), bound, what)
