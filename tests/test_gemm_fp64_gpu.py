"""GPU: yamb_pointwise_gemm called directly for every case of tests/gemm_cases.py, every output
compared with a float64 reference of the same operation, element by element.

Operands.  The reference first forms the bf16 operands the kernel feeds to wgmma, in the kernel's
order of operations: mode 1 z = fmaf(s, x, b) (the sum formed in fp64, rounded once to fp32), then
the clamp or activation, then RN to bf16, and with an SE gate RN_bf16(RN_bf16(act(z)) * gate);
mode 2 fmaf(s, x, fmaf(s2, x2, b)) then RN to bf16.  With no activation, ReLU or ReLU6 these are
exact.  Swish and h-swish run on fp32 intrinsics: an element within 2^-16 of a bf16 rounding
boundary may be one ulp off; that ulp (da, db) enters the bound as sum da |b| + |a| db.

Outputs.  With S = |A'| @ |B'|^T in fp64:
  epi 0 / 1: D must lie between the bf16 values of ref -+ E, E = 2^-22 (ceil(K/16) + 2) S (+ the
             fp32 add of the residual, + act' of the intrinsics for epi 1);
  epi 2:     |D - (D0 + ref)| <= E + 2^-23 (ksplit + 1) (S + |D0|) against a nonzero prefilled D0
             (the split-K slabs are added in fp32, then added to D0).
E allows two fp32 ulps of the running magnitude per 16-wide wgmma k-step (Hopper's accumulation
order inside a step is not documented; the rule passes on an H100 and, below, is shown to be
tight enough to see one missing k-step).  Every case drops one 16-wide k-step, chosen at random,
from the fp64 reference and requires the checker to flag at least 90 % of the elements it changes.

Statistics are fp64 sums over the D the kernel stored (sum h and sum h^2 for epi 0; sum dz and
sum dz * xhat for epi 1 with xhat = fmaf(h, r, -m r) in fp32), bound 2^-24 (L + 2) sum |term|
with L the longest fp32 chain of the plan: 8 rows per interleaved chain + 2 to combine the four
chains + the tiles each warp adds into its register sums (reg_stats), or 1.  Derived values carry
the propagated bound (tests/ref64.py); running statistics are checked against nn.BatchNorm2d.

Every call also checks: the BatchNorm accumulator and counter come back zero; a second identical
call gives identical bits; for epi 0 / 1 D has the same bits at max_ctas 1, 2 and 5 as at the
default grid (for epi 2 where ksplit is the same); sentinels survive outside the channel slice, in
the row after M and in the pitch padding; a poison row after the last row of every input and NaN
between the row length and the pitch reach no output.  On failure the message names the element
and, from the library's plan, its m / n-block, tile, CTA and walk step."""
import ctypes as C
import math

import pytest
import torch

import gemm_cases as gc
from ref64 import (BAND, DEV, POISON, SENTINEL, _Acc, _act64, _bwd_outputs, _bn_bwd,
                   _check_bwd_finalize, _check_fwd_finalize, _check_guard, _clamp32, _dact64,
                   _act_err, _eval_mode_coeffs, _f32, _guarded, _outside, _same, _worst)

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
NAN = float("nan")


def _nat():
    from yet_another_mobilenet_series_b200 import native as nat
    return nat


def _plan(lib, c, max_ctas=None):
    nat = _nat()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rc, info = gc.plan(lib, nat, c, sms=sms, max_ctas=max_ctas)
    assert rc == 0, lib.yamb_last_error()
    return info


def _loc(c, p):
    def loc(row, col, *_):
        m_blk, n_blk = row // 128, col // p.block_n
        mn = m_blk * p.n_blocks + n_blk
        ws = [mn * p.ksplit + s for s in range(p.ksplit)]
        where = ", ".join("slab %d: CTA %d step %d" % (s, w % p.grid, w // p.grid)
                          for s, w in enumerate(ws[:4]))
        return "(row %d, column %d: m-block %d, n-block %d, tile %d; %s; grid %d)" % (
            row, col, m_blk, n_blk, mn, where, p.grid)
    return loc


# ---- operands --------------------------------------------------------------------------------------
def _stored(vals, ld, fill=NAN):
    """[rows, cols] values -> [rows + 1, ld] buffer: NaN between cols and ld, a poison last row."""
    rows, cols = vals.shape
    buf = torch.full((rows + 1, ld), fill, device=DEV, dtype=vals.dtype)
    buf[:rows, :cols] = vals
    buf[rows, :cols] = POISON
    return buf


def _xform(x, mode, act, s, b, s2=None, x2=None, gate_rows=None):
    """Operand the kernel feeds to wgmma, in the stored orientation [pixels, channels]:
    (value fp64, one-ulp band fp64)."""
    x64 = x.double()
    if mode == 2:
        t1 = _f32(x2.double() * s2.double() + b.double())
        v = _f32(x64 * s.double() + t1.double()).to(BF).double()
        return v, torch.zeros_like(v)
    z32 = _f32(x64 * s.double() + b.double())

    def gated(a32):
        a = a32.to(BF)
        if gate_rows is not None:
            a = _f32(a.double() * gate_rows.double()).to(BF)
        return a.double()

    if act in (0, 1, 2):
        v = gated(_clamp32(z32, act))
        return v, torch.zeros_like(v)
    a64 = _act64(z32, act)
    lo, hi = gated((a64 * (1 - BAND)).float()), gated((a64 * (1 + BAND)).float())
    return gated(a64.float()), (hi - lo).abs()


class _Data:
    """Inputs of one case (stored buffers) and the fp64 operands A' [M, K], B' [N, K]."""

    def __init__(self, c, gen):
        M, N, K = c.M, c.N, c.K
        p = gc.pitches(c)
        self.c, self.keep = c, {}
        self.ptrs = {}
        for side in ("a", "b"):
            mn = c.a_mn if side == "a" else c.b_mn
            xf = c.a_xform if side == "a" else c.b_xform
            rows = K if mn else (M if side == "a" else N)
            ch = (M if side == "a" else N) if mn else K
            ld = p["lda" if side == "a" else "ldb"]
            if xf:
                x = (torch.randn(rows, ch, device=DEV, generator=gen) * 1.5 + 0.3).to(BF)
            elif side == "a":
                x = torch.randn(rows, ch, device=DEV, generator=gen).to(BF)
            else:
                x = (torch.randn(rows, ch, device=DEV, generator=gen) / math.sqrt(K)).to(BF)
            if c.shifted:      # a constant channel: D's column means ~8x their spread
                if side == "a":
                    x[:, 0] = 1.0
                else:
                    x[:, 0] = 8.0 * (torch.randint(0, 2, (rows,), device=DEV, generator=gen) * 2 - 1)
            buf = _stored(x, ld)
            self.keep[side.upper()] = buf
            self.ptrs[side.upper()] = buf.data_ptr()
            if xf:
                s = torch.rand(ch, device=DEV, generator=gen) + 0.5
                b = torch.randn(ch, device=DEV, generator=gen) * 0.3
                s2 = x2 = grows = None
                if xf == 2:
                    s2 = torch.randn(ch, device=DEV, generator=gen) * 0.5
                    x2 = torch.randn(rows, ch, device=DEV, generator=gen).to(BF)
                    b2 = _stored(x2, ld)
                    self.keep[side.upper() + "2"] = b2
                    self.ptrs[side.upper() + "2"] = b2.data_ptr()
                    self.ptrs[side + "_scale2"] = s2.data_ptr()
                if c.gate and xf == 1:
                    nsamp = -(-rows // c.gate)
                    gate = torch.rand(nsamp, ch, device=DEV, generator=gen) + 0.25
                    self.keep["gate"] = gate
                    self.ptrs["gate"] = gate.data_ptr()
                    grows = gate[torch.arange(rows, device=DEV) // c.gate]
                self.keep[side + "_sb"] = (s, b, s2)
                self.ptrs[side + "_scale"], self.ptrs[side + "_shift"] = s.data_ptr(), b.data_ptr()
                v, d = _xform(x, xf, c.act, s, b, s2, x2, grows)
                del grows
            else:
                v, d = x.double(), None
            if mn:
                v = v.t()
                d = None if d is None else d.t()
            setattr(self, side + "64", v)
            setattr(self, "d" + side, d)
        lds = p["lds"]
        if c.residual:
            r = torch.randn(M, N, device=DEV, generator=gen).to(BF)
            self.R = _stored_slice(r, c.c0, lds)
            self.ptrs["residual"] = self.R.data_ptr() + 2 * c.c0
        if c.epi == 1:
            self.H = _stored_slice((torch.randn(M, N, device=DEV, generator=gen) * 1.5).to(BF),
                                   c.c0, lds)
            self.hs = torch.rand(N, device=DEV, generator=gen) + 0.5
            self.ht = torch.randn(N, device=DEV, generator=gen) * 0.3
            self.ptrs["H"] = self.H.data_ptr() + 2 * c.c0
            self.ptrs["h_scale"], self.ptrs["h_shift"] = self.hs.data_ptr(), self.ht.data_ptr()
        if c.epi == 2:
            self.D0 = torch.randn(M, N, device=DEV, generator=gen) * 0.5


def _stored_slice(vals, c0, ld):
    """[M, N] -> [M + 1, ld] with vals at columns c0.., NaN elsewhere, a poison last row."""
    M, N = vals.shape
    buf = torch.full((M + 1, ld), NAN, device=DEV, dtype=vals.dtype)
    buf[:M, c0:c0 + N] = vals
    buf[M, :] = POISON
    return buf


# ---- one call ------------------------------------------------------------------------------------
class _Bn:
    """BatchNorm structs and their (guarded) outputs for one call."""

    def __init__(self, c, data, gen):
        N = c.N
        self.acc = _Acc(N)
        if c.epi == 0 and c.stats:
            self.gamma = torch.rand(N, device=DEV, generator=gen) + 0.5 if c.affine else None
            self.beta = torch.randn(N, device=DEV, generator=gen) if c.affine else None
            self.rm0 = torch.randn(N, device=DEV, generator=gen) * 0.1
            self.rv0 = torch.rand(N, device=DEV, generator=gen) + 0.5
            self.nbt0 = 3
        if c.epi == 1:
            h64 = data.H[:c.M, c.c0:c.c0 + N].double()
            self.gamma = torch.rand(N, device=DEV, generator=gen) + 0.5 if c.affine else None
            self.mean1 = _f32(h64.mean(0))
            self.invstd1 = _f32((h64.var(0, unbiased=False) + 1e-3).rsqrt())
            self.dg0 = torch.randn(N, device=DEV, generator=gen) * 10
            self.db0 = torch.randn(N, device=DEV, generator=gen) * 10

    def fwd(self, nat, c, momentum=None, o_prev=None):
        N = c.N
        o = {k: _guarded(N) for k in ("scale", "shift")}
        if c.running:
            o["mean"], o["invstd"] = _guarded(N), _guarded(N)
            o["rm"], o["rv"] = _guarded(N), _guarded(N)
            src = o_prev if o_prev is not None else {"rm": self.rm0, "rv": self.rv0}
            o["rm"][:N], o["rv"][:N] = src["rm"][:N], src["rv"][:N]
            o["nbt"] = torch.full((1,), self.nbt0, device=DEV, dtype=torch.int64) \
                if o_prev is None else o_prev["nbt"].clone()
        f = nat.BnFwd()
        f.partials, f.counter = self.acc.partials.data_ptr(), self.acc.counter.data_ptr()
        f.gamma = None if self.gamma is None else self.gamma.data_ptr()
        f.beta = None if self.beta is None else self.beta.data_ptr()
        mom = c.mom if momentum is None else momentum
        f.eps, f.momentum = 1e-3, -1.0 if mom is None else mom
        if c.running:
            f.running_mean, f.running_var = o["rm"].data_ptr(), o["rv"].data_ptr()
            f.num_batches_tracked = o["nbt"].data_ptr()
            f.mean, f.invstd = o["mean"].data_ptr(), o["invstd"].data_ptr()
        f.scale, f.shift = o["scale"].data_ptr(), o["shift"].data_ptr()
        f.count = c.M
        return f, o

    def bwd(self, c, use_batch_stats=None):
        out = _bwd_outputs(c.N, self.dg0, self.db0)
        if not c.grads:
            out["dg"] = out["db"] = None
        ubs = c.use_batch_stats if use_batch_stats is None else use_batch_stats
        return _bn_bwd(self.acc, c.N, c.M, self.gamma, self.mean1, self.invstd1, out, ubs), out


def _run(lib, c, data, bn, max_ctas=None, stream=None, use_batch_stats=None, o_prev=None):
    """One call; returns (D buffer, BatchNorm outputs)."""
    nat = _nat()
    p = gc.pitches(c)
    if c.epi == 2:
        D = torch.full((c.M + 1, p["ldd"]), SENTINEL, device=DEV, dtype=torch.float32)
        D[:c.M, c.c0:c.c0 + c.N] = data.D0
    else:
        D = torch.full((c.M + 1, p["ldd"]), SENTINEL, device=DEV, dtype=BF)
    ptrs = dict(data.ptrs)
    ptrs["D"] = D.data_ptr() + D.element_size() * c.c0
    g = gc.gemm_struct(nat, c, ptrs, max_ctas)
    o = None
    if c.epi == 0 and c.stats:
        f, o = bn.fwd(nat, c, o_prev=o_prev)
        g.bn_fwd = C.pointer(f)
    if c.epi == 1:
        b, o = bn.bwd(c, use_batch_stats)
        g.bn_bwd = C.pointer(b)
    s = stream.cuda_stream if stream is not None else nat.stream_handle()
    nat.check(lib.yamb_pointwise_gemm(C.byref(g), s))
    if stream is None:
        bn.acc.check()
    return D, o


# ---- reference -----------------------------------------------------------------------------------
def _reference(c, data, r0, r1, drop=None):
    """fp64 reference of output rows [r0, r1) before the output rounding: (y, E, S).  drop: a
    k-step left out of the reference."""
    a, b = data.a64[r0:r1], data.b64
    ref = a @ b.t()
    mag = a.abs() @ b.abs().t()
    if drop is not None:
        k0 = drop * 16
        ref = ref - a[:, k0:k0 + 16] @ b[:, k0:k0 + 16].t()
    E = 2.0 ** -22 * (-(-c.K // 16) + 2) * mag
    if data.da is not None:
        E += data.da[r0:r1] @ b.abs().t()
    if data.db is not None:
        E += a.abs() @ data.db.t()
    if c.epi == 0 and c.residual:
        r = data.R[r0:r1, c.c0:c.c0 + c.N].double()
        E += 2.0 ** -23 * (ref.abs() + r.abs() + E)
        ref = ref + r
    if c.epi == 1:
        h = data.H[r0:r1, c.c0:c.c0 + c.N].double()
        z32 = _f32(h * data.hs.double() + data.ht.double())
        gp = _dact64(z32, c.act)
        E = E * gp.abs() + (ref.abs() + E) * _act_err(z32.double(), c.act, gp)
        ref = ref * gp
        E += 2.0 ** -23 * ref.abs()     # the fp32 product before the bf16 rounding
    return ref, E, mag


def _check_output(c, data, D, p, gen):
    """Every element against the fp64 reference; and the reference without one k-step must fail."""
    loc = _loc(c, p)
    got_all = D[:c.M, c.c0:c.c0 + c.N]
    steps = -(-c.K // 16)
    drop = int(torch.randint(0, steps, (1,), device=DEV, generator=gen))
    touched = flagged = 0
    rows = c.M if c.epi == 2 else gc.REF_ROWS
    for r0 in range(0, c.M, rows):
        r1 = min(c.M, r0 + rows)
        got = got_all[r0:r1]
        y, E, S = _reference(c, data, r0, r1)
        yd = _reference(c, data, r0, r1, drop)[0]
        if c.epi == 2:
            D0 = data.D0[r0:r1].double()
            E = E + 2.0 ** -23 * (p.ksplit + 1) * (S + D0.abs())
            err = (got.double() - D0 - y).abs()
            assert bool(torch.isfinite(got).all()), "epi 2: non-finite output"
            _worst(err, E, "D", lambda i, j: loc(i + r0, j))
            bad_d = (got.double() - D0 - yd).abs() > E
            ch = (yd - y) != 0
        else:
            bad, lo, hi = _outside(got, y, E)
            if bool(bad.any()):
                i = int(bad.flatten().nonzero()[0])
                ri, ci = divmod(i, c.N)
                raise AssertionError("D: got %r outside [%r, %r] (exact %r; %d elements) %s" % (
                    float(got[ri, ci]), float(lo[ri, ci]), float(hi[ri, ci]), float(y[ri, ci]),
                    int(bad.sum()), loc(ri + r0, ci)))
            bad_d = _outside(got, yd, E)[0]
            ch = (yd - y) != 0
        touched += int(ch.sum())
        flagged += int((bad_d & ch).sum())
        del y, E, yd, S
    assert touched > 0
    frac = flagged / touched
    assert frac >= 0.9, "the bound does not see k-step %d missing: %.1f%% of %d elements flagged" % (
        drop, 100 * frac, touched)


def _chain(c, p):
    """Longest fp32 chain of the column statistics (see the module docstring)."""
    return 8 + 2 + (gc.tiles_per_cta(p) if p.reg_stats else 1)


def _check_frame(D, c, what):
    ldd = D.shape[1]
    ok = bool((D[:c.M, :c.c0] == SENTINEL).all()) and bool((D[:c.M, c.c0 + c.N:] == SENTINEL).all())
    assert ok, "%s: wrote columns outside [%d, %d) of the pitch %d" % (what, c.c0, c.c0 + c.N, ldd)
    assert bool((D[c.M] == SENTINEL).all()), "%s: wrote the row after M" % what


# ================================================================================================
@pytest.mark.parametrize("name", [c.name for c in gc.CASES])
def test_gemm_fp64(built_lib, name):
    c = gc.BY_NAME[name]
    lib = built_lib
    gen = torch.Generator(device=DEV).manual_seed(1000 + c.seed + gc.CASES.index(c))
    data = _Data(c, gen)
    bn = _Bn(c, data, gen)
    p = _plan(lib, c)
    D, o = _run(lib, c, data, bn)
    torch.cuda.synchronize()
    _check_frame(D, c, name)
    # a second identical call: identical bits (D and every BatchNorm output)
    D2, o2 = _run(lib, c, data, bn, o_prev=None)
    _same(D, D2, name + " D")
    if o is not None:
        for k in o:
            if o[k] is not None:
                _same(o[k], o2[k], name + " " + k)
    del D2
    # other grids: the same bits (epi 2: where ksplit is the same)
    for mc in (1, 2, 5):
        q = _plan(lib, c, max_ctas=mc)
        if c.epi == 2 and q.ksplit != p.ksplit:
            continue
        Dm, _ = _run(lib, c, data, bn, max_ctas=mc)
        _same(Dm, D, "%s D at max_ctas %d (grid %d) vs grid %d" % (name, mc, q.grid, p.grid))
        del Dm
    torch.cuda.synchronize()
    _check_output(c, data, D, p, gen)
    data.a64 = data.da = None      # the fp64 operands are not needed any more
    loc = _loc(c, p)
    chan = lambda j, *_: loc(0, j)
    if c.epi == 0 and c.stats:
        h64 = D[:c.M, c.c0:c.c0 + c.N].double()
        t = 2.0 ** -24 * (_chain(c, p) + 2)
        b_s, b_q = t * h64.abs().sum(0), t * (h64 * h64).sum(0)
        if not c.running:
            o["rm"] = o["nbt"] = None
        mean_ref, var_ref, inv_ref = _check_fwd_finalize(
            o, h64, bn.gamma, bn.beta, bn.rm0, bn.rv0, bn.nbt0, 1e-3, c.mom, b_s, b_q, name, chan)
        for k in o:
            if o[k] is not None and k != "nbt":
                _check_guard(o[k], c.N, name + " " + k)
        if c.shifted:
            ratio = float((mean_ref.abs() / var_ref.sqrt()).median())
            e_inv = (o["invstd"][:c.N].double() - inv_ref).abs()
            lo = (var_ref + 1e-3 - b_q / c.M - 2 * mean_ref.abs() * b_s / c.M).clamp_min(1e-300)
            bound = 0.5 * (b_q / c.M + 2 * mean_ref.abs() * b_s / c.M) * lo ** -1.5 + \
                2.0 ** -23 * inv_ref
            print("\nlong chain: %d rows, %d tiles per CTA, median |mean|/std %.1f; invstd max rel "
                  "err %.2e, its bound %.2e" % (c.M, gc.tiles_per_cta(p), ratio,
                                                float((e_inv / inv_ref).max()),
                                                float((bound / inv_ref).max())))
            assert ratio > 6.0
        if c.running:
            # a second call from the first one's running statistics (momentum=None: the
            # cumulative factor moves on with num_batches_tracked)
            _, o3 = _run(lib, c, data, bn, o_prev=o)
            _check_fwd_finalize(o3, h64, bn.gamma, bn.beta, o["rm"][:c.N], o["rv"][:c.N],
                                bn.nbt0 + 1, 1e-3, c.mom, b_s, b_q, name + " (second call)", chan)
    if c.epi == 1:
        dz = D[:c.M, c.c0:c.c0 + c.N].double()
        h = data.H[:c.M, c.c0:c.c0 + c.N].double()
        r = bn.invstd1.double()
        nmr = _f32(-bn.mean1.double() * r).double()
        xhat = _f32(h * r + nmr).double()
        t = 2.0 ** -24 * (_chain(c, p) + 2)
        s_ref, q_ref = dz.sum(0), (dz * xhat).sum(0)
        b_s, b_q = t * dz.abs().sum(0), t * (dz * xhat).abs().sum(0)
        # use_batch_stats = 0 cases: dgamma / dbeta / ca from a train-mode call, then the
        # eval-mode coefficients against it
        o1 = o if c.use_batch_stats else _run(lib, c, data, bn, use_batch_stats=1)[1]
        _check_bwd_finalize(o1, c.N, c.M, bn.gamma, bn.mean1, bn.invstd1, s_ref, q_ref, b_s, b_q,
                            bn.dg0, bn.db0, name, chan)
        _eval_mode_coeffs(lambda u: _run(lib, c, data, bn, use_batch_stats=u)[1], o1, c.N,
                          bn.gamma, bn.invstd1, name)


# ---- act' at the edges of the dz epilogue -------------------------------------------------------
_EDGES = [0.0, 6.0, -3.0, 3.0]
_POINTS = _EDGES + [-6.0, -1.0, 1.0, 5.5, 6.5, -2.5, 2.5, 0.5]


@pytest.mark.parametrize("act", [1, 2, 3, 4])
def test_dz_activation_edges(built_lib, act):
    """H exactly 0, 6, -3, +3 (scale 1, shift 0): dz = RN(acc * act'(z)) with act' from fp64
    autograd through nn.ReLU / nn.ReLU6 / Swish / HSwish (0 at both ReLU6 edges and ReLU's 0,
    0 at h-swish -3, 1 at +3, 1/2 at h-swish 0)."""
    nat = _nat()
    c = gc.Case("edges", 256, 64, 16, b_mn=1, epi=1, act=act)
    gen = torch.Generator(device=DEV).manual_seed(20 + act)
    data = _Data(c, gen)
    pts = torch.tensor(_POINTS, device=DEV)
    idx = (torch.arange(c.M, device=DEV)[:, None] + torch.arange(c.N, device=DEV)[None, :]) % len(pts)
    data.H[:c.M, :c.N] = pts[idx].to(BF)
    data.hs.fill_(1.0)
    data.ht.fill_(0.0)
    bn = _Bn(c, data, gen)
    D, _ = _run(built_lib, c, data, bn)
    torch.cuda.synchronize()
    ref = data.a64 @ data.b64.t()
    hz = data.H[:c.M, :c.N].double()
    gp = _dact64(hz, act)
    for e, v in {1: {0.0: 0, 6.0: 1, -3.0: 0, 3.0: 1}, 2: {0.0: 0, 6.0: 0, -3.0: 0, 3.0: 1},
                 4: {0.0: 0.5, 6.0: 1, -3.0: 0, 3.0: 1}}.get(act, {}).items():
        assert bool((gp[hz == e] == v).all()), ("reference derivative", act, e)
    edge = torch.zeros_like(hz, dtype=torch.bool)
    for e in (_EDGES if act != 3 else [0.0]):
        edge |= hz == e
    got = D[:c.M, :c.N].double()
    E = 2.0 ** -22 * 3 * (data.a64.abs() @ data.b64.abs().t())
    bad, _, _ = _outside(got[edge], (ref * gp)[edge], (E * gp.abs())[edge])
    assert not bool(bad.any()), "act' at the edges: %d elements" % int(bad.sum())
    # at an edge where act' is 0 the output is exactly 0
    z = edge & (gp == 0)
    assert bool((got[z] == 0).all())


# ---- concurrency ---------------------------------------------------------------------------------
def test_wgrad_side_stream_with_dgrad(built_lib):
    """A project wgrad (epi 2) on a side stream and a dgrad (epi 1) on the main stream at the same
    time give the bits each gives alone (the engine's side-stream pattern)."""
    cw, cd = gc.BY_NAME["wgrad_big"], gc.BY_NAME["dz_swish_multi"]
    gen = torch.Generator(device=DEV).manual_seed(31)
    dw, dd = _Data(cw, gen), _Data(cd, gen)
    bw, bd = _Bn(cw, dw, gen), _Bn(cd, dd, gen)
    Dw, _ = _run(built_lib, cw, dw, bw)
    Dd, od = _run(built_lib, cd, dd, bd)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    for _ in range(3):
        with torch.cuda.stream(side):
            Dw2, _ = _run(built_lib, cw, dw, bw, stream=side)
        Dd2, od2 = _run(built_lib, cd, dd, bd)
        torch.cuda.synchronize()
        _same(Dw2, Dw, "side-stream wgrad")
        _same(Dd2, Dd, "main-stream dgrad")
        for k in ("ca", "cb", "cc"):
            _same(od2[k], od[k], "main-stream dgrad " + k)


# ---- refusals ------------------------------------------------------------------------------------
def test_refusals_leave_outputs_untouched(built_lib):
    """Malformed calls return YAMB_EINVAL with a message, write nothing (D, the BatchNorm counter
    and accumulator), and a valid call right afterwards succeeds."""
    nat = _nat()
    c = gc.BY_NAME["fwd_slice_stats"]
    gen = torch.Generator(device=DEV).manual_seed(41)
    data = _Data(c, gen)
    bn = _Bn(c, data, gen)
    p = gc.pitches(c)
    D = torch.full((c.M + 1, p["ldd"]), SENTINEL, device=DEV, dtype=BF)

    def call(edit):
        ptrs = dict(data.ptrs, D=D.data_ptr() + 2 * c.c0)
        g = gc.gemm_struct(nat, c, ptrs)
        f, _ = bn.fwd(nat, c)
        g.bn_fwd = C.pointer(f)
        edit(g)
        return built_lib.yamb_pointwise_gemm(C.byref(g), nat.stream_handle())

    bad = {
        "A offset by 2 bytes": lambda g: setattr(g, "A", g.A + 2),
        "B offset by 2 bytes": lambda g: setattr(g, "B", g.B + 2),
        "D offset by 2 bytes": lambda g: setattr(g, "D", g.D + 2),
        "lda % 8": lambda g: setattr(g, "lda", g.lda + 4),
        "ldb % 8": lambda g: setattr(g, "ldb", g.ldb + 2),
        "ldd % 8": lambda g: setattr(g, "ldd", g.ldd + 4),
        "N % 8": lambda g: setattr(g, "N", 44),
        "layout": lambda g: setattr(g, "a_mn_major", 1),
        "no A": lambda g: setattr(g, "A", None),
    }
    for what, edit in bad.items():
        rc = call(edit)
        assert rc == -1 and built_lib.yamb_last_error() != b"", (what, rc)
        torch.cuda.synchronize()
        assert bool((D == SENTINEL).all()), what + ": D written"
        bn.acc.check()
    assert call(lambda g: None) == 0
    bn.acc.check()
    assert not bool((D[:c.M, c.c0:c.c0 + c.N] == SENTINEL).any())
