"""The one-launch eval block (csrc/block_eval.cuh) element by element against fp64 with rounding
intervals (tests/block_eval_ref64.py), on every compiled (tile geometry, expansion, activation
class) in the plain, gate and pool modes, unsplit and split over a thread-block cluster
(tests/block_eval_cases.py; tests/test_block_eval_plan_cpu.py pins that the table reaches them).

Three probes per case, through the C ABI:
  * expand: one-hot depthwise taps (centre, edges and corners), BatchNorms 2 and 3 identities
    (gamma / beta NULL, mean 0, var = eps = 0.5), a project that selects one hidden channel per
    output column (the first and last channel of every 64-channel slice among them), no residual:
    y[n, j, o] = act(a1[n, c_j, o * S + tap - P]), 0 outside the image.  A bit-exact view of the
    expand MMA, BatchNorm 1 and the halo;
  * stencil: random depthwise weights and BatchNorms 1 / 2, the same selecting project: y = a2
    (a2s with the gate);
  * full: everything random, the residual where the case has one, and the pool pass.
The split launch must give the unsplit bits wherever an output is a single exact term (expand and
stencil probes) and for the pooled means.  y and pooled are followed by 8 guard values that must
keep ref64.SENTINEL."""
import ctypes as C

import pytest
import torch

import block_eval_cases as bc
import block_eval_ref64 as br
import ref64

pytestmark = pytest.mark.gpu
DEV = "cuda"
PROBES = ("expand", "stencil", "full")


def _taps(k):
    p, e = (k - 1) // 2, k - 1
    return [(p, p), (0, p), (e, p), (p, 0), (p, e), (0, 0), (0, e), (e, 0), (e, e)]


def _selection(Chid, Cout):
    """Hidden channel of every output column: the first and last of every 64-channel slice, then
    a stride through the rest."""
    sel = []
    for s in range(0, Chid, 64):
        for c in (s, min(s + 63, Chid - 1)):
            if c not in sel:
                sel.append(c)
    j = 0
    while len(sel) < Cout:
        sel.append((7 + 37 * j) % Chid)
        j += 1
    return sel[:Cout]


def _bn(C, affine, gen, eps):
    u = lambda a, b: torch.rand(C, generator=gen, device=DEV) * (b - a) + a
    sign = torch.where(torch.rand(C, generator=gen, device=DEV) < 0.2, -1.0, 1.0)
    return {"gamma": u(0.5, 1.5) * sign if affine else None,
            "beta": torch.randn(C, generator=gen, device=DEV) * 0.3 if affine else None,
            "mean": torch.randn(C, generator=gen, device=DEV) * 0.5, "var": u(0.5, 2.0), "eps": eps}


def _identity_bn(C):
    return {"gamma": None, "beta": None, "mean": torch.zeros(C, device=DEV),
            "var": torch.full((C,), 0.5, device=DEV), "eps": 0.5}


def _params(c, probe, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    k = c.k
    x = torch.randn(c.N, c.Cin, c.H, c.W, generator=gen, device=DEV).bfloat16()
    w1 = (torch.randn(c.Chid, c.Cin, generator=gen, device=DEV) * (2.0 / c.Cin) ** 0.5).bfloat16()
    sel = _selection(c.Chid, c.Cout)
    if probe == "full":
        w3 = (torch.randn(c.Cout, c.Chid, generator=gen, device=DEV) * (1.0 / c.Chid) ** 0.5).bfloat16()
    else:
        w3 = torch.zeros(c.Cout, c.Chid, device=DEV)
        w3[torch.arange(c.Cout, device=DEV), torch.tensor(sel, device=DEV)] = 1.0
        w3 = w3.bfloat16()
    if probe == "expand":
        wdw = torch.zeros(c.Chid, k * k, device=DEV)
        taps = _taps(k)
        for ch in range(c.Chid):
            ky, kx = taps[ch % len(taps)]
            wdw[ch, ky * k + kx] = 1.0
    else:
        wdw = torch.randn(c.Chid, k * k, generator=gen, device=DEV) * (2.0 / (k * k)) ** 0.5
    bn1 = _bn(c.Chid, c.affine, gen, 1e-3)
    if probe == "expand":
        bn2, bn3 = _identity_bn(c.Chid), _identity_bn(c.Cout)
    else:
        bn2 = _bn(c.Chid, c.affine, gen, 1e-5)
        bn3 = _bn(c.Cout, c.affine, gen, 0.1) if probe == "full" else _identity_bn(c.Cout)
    gate = torch.rand(c.N, c.Chid, generator=gen, device=DEV) * 1.5
    residual = c.residual and probe == "full"
    return dict(x=x, w1=w1, wdw=wdw, w3=w3, bn1=bn1, bn2=bn2, bn3=bn3, gate=gate, residual=residual)


def _reference(c, P):
    x = P["x"].double()
    if c.expand:
        a1 = br.expand(x, P["w1"], P["bn1"], c.act)
    else:
        a1 = (x, x)
    a2 = br.stencil(*a1, P["wdw"], c.k, c.s, P["bn2"], c.act)
    res = x if P["residual"] else None
    ref = {"a2": a2,
           "y": br.project(*a2, P["w3"], P["bn3"], res, extra_adds=8),
           "y_gate": br.project(*br.gated(*a2, P["gate"]), P["w3"], P["bn3"], res, extra_adds=8)}
    g, _, _ = bc.case_plan(c)
    nslab = bc._cdiv(a2[0].shape[2], g.toh) * bc._cdiv(a2[0].shape[3], g.tow)
    ref["pooled"] = br.pooled(*a2, nslab)
    return ref


def _bn_struct(dst, bn):
    if bn is None:
        return
    dst.gamma = ref64._nat().ptr(bn["gamma"])
    dst.beta = ref64._nat().ptr(bn["beta"])
    dst.running_mean = bn["mean"].data_ptr()
    dst.running_var = bn["var"].data_ptr()
    dst.eps = bn["eps"]


def _launch(lib, c, P, x_nhwc, mode, cs):
    """One call of the C ABI; returns the guarded output (y [N*Ho*Wo*Cout + 8] bf16 or pooled
    [N*Chid + 8] fp32)."""
    nat = ref64._nat()
    Ho, Wo = bc.out_size(c.H, c.s), bc.out_size(c.W, c.s)
    a = nat.BlockEval()
    a.N, a.H, a.W, a.Cin, a.Chid, a.Cout = c.N, c.H, c.W, c.Cin, c.Chid, c.Cout
    a.kernel, a.stride, a.act, a.residual = c.k, c.s, c.act, 1 if P["residual"] else 0
    a.x = x_nhwc.data_ptr()
    a.w_expand = P["w1"].data_ptr() if c.expand else None
    a.w_dw = P["wdw"].data_ptr()
    a.w_project = P["w3"].data_ptr()
    _bn_struct(a.bn1, P["bn1"] if c.expand else None)
    _bn_struct(a.bn2, P["bn2"])
    _bn_struct(a.bn3, P["bn3"])
    st = torch.cuda.current_stream().cuda_stream
    if mode == "pool":
        out = ref64._guarded(c.N * c.Chid, fill=float("nan"))
        a.pooled = out.data_ptr()
        rc = lib.yamb_block_eval_pool_fwd(C.byref(a), st) if cs == 1 else \
            lib.yamb_block_eval_cluster_pool_fwd(C.byref(a), cs, st)
    else:
        out = ref64._guarded(c.N * Ho * Wo * c.Cout, fill=ref64.SENTINEL, dtype=torch.bfloat16)
        a.y = out.data_ptr()
        a.gate = P["gate"].data_ptr() if mode == "gate" else None
        rc = lib.yamb_block_eval_fwd(C.byref(a), st) if cs == 1 else \
            lib.yamb_block_eval_cluster_fwd(C.byref(a), cs, st)
    assert rc == 0, (c.name, mode, cs, lib.yamb_last_error())
    torch.cuda.synchronize()
    return out


def _locator(c):
    g, _, _ = bc.case_plan(c)
    Ho, Wo = bc.out_size(c.H, c.s), bc.out_size(c.W, c.s)
    tw, th = bc._cdiv(Wo, g.tow), bc._cdiv(Ho, g.toh)

    def loc(n, j, oy, ox):
        t = ((n // g.ti) * th + oy // g.toh) * tw + ox // g.tow
        return "(n, column, oy, ox); tile %d of %d at row %d, col %d of the tile" % (
            t, th * tw * bc._cdiv(c.N, g.ti), oy % g.toh, ox % g.tow)
    return loc


def _check_y(c, out, lo, hi, what):
    Ho, Wo = bc.out_size(c.H, c.s), bc.out_size(c.W, c.s)
    n = c.N * Ho * Wo * c.Cout
    ref64._check_guard(out, n, what)
    y = out[:n].view(c.N, Ho, Wo, c.Cout).permute(0, 3, 1, 2).double()
    bad = (y < lo) | (y > hi) | ~torch.isfinite(y)
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), bad.shape))
        ref64._fail(what, idx, _locator(c), "got %r outside [%r, %r] (%d elements)" % (
            float(y[idx]), float(lo[idx]), float(hi[idx]), int(bad.sum())))
    return out[:n]


def _width(lo, hi):
    return float((br.count_values(lo, hi) > 2).double().mean())


@pytest.mark.parametrize("case", bc.CASES, ids=[c.name for c in bc.CASES])
def test_block_eval_fp64(built_lib, case):
    c = case
    widths = []
    for pi, probe in enumerate(PROBES):
        P = _params(c, probe, 1000 + 7 * pi + sum(c[1:7]))
        ref = _reference(c, P)
        x_nhwc = P["x"].permute(0, 2, 3, 1).contiguous()
        modes = ("plain",) if probe == "expand" else ("plain", "gate")
        for mode in modes:
            lo, hi = ref["y" if mode == "plain" else "y_gate"]
            widths.append("%s/%s %.2e" % (probe, mode, _width(lo, hi)))
            ys = {}
            for cs in (1, c.cs):
                what = "%s: %s probe, %s, cluster %d" % (c.name, probe, mode, cs)
                ys[cs] = _check_y(c, _launch(built_lib, c, P, x_nhwc, mode, cs), lo, hi, what)
            if probe != "full":
                ref64._same(ys[1], ys[c.cs], "%s: %s probe, %s, cluster %d vs unsplit"
                            % (c.name, probe, mode, c.cs))
        if probe == "full":
            plo, phi = ref["pooled"]
            pools = {}
            for cs in (1, c.cs):
                what = "%s: pool pass, cluster %d" % (c.name, cs)
                out = _launch(built_lib, c, P, x_nhwc, "pool", cs)
                ref64._check_guard(out, c.N * c.Chid, what)
                got = out[:c.N * c.Chid].view(c.N, c.Chid).double()
                bad = (got < plo) | (got > phi) | ~torch.isfinite(got)
                if bool(bad.any()):
                    i = int(bad.flatten().nonzero()[0])
                    n, ch = divmod(i, c.Chid)
                    raise AssertionError("%s: pooled[%d][%d] = %r outside [%r, %r] (%d elements)" % (
                        what, n, ch, float(got[n, ch]), float(plo[n, ch]), float(phi[n, ch]),
                        int(bad.sum())))
                pools[cs] = out
            ref64._same(pools[1], pools[c.cs], "%s: pooled, cluster %d vs unsplit" % (c.name, c.cs))
    g, ex, nt = bc.case_plan(c)
    print("%-24s %s tiles %4d  intervals of > 2 bf16 values: %s"
          % (c.name, tuple(g), nt, ", ".join(widths)))
