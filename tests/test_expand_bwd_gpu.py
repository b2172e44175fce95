"""yamb_expand_bwd (csrc/expand_bwd.cu) on the GPU: every instantiation (wgmma width 16 / 32 x one,
two or three 64-channel panels) against float64, element by element; dx and dW1 bit for bit
against the dgrad and split-K wgrad GEMMs, also when a slab ends inside a 128-pixel unit; dW1
accumulates; repeated and graph-replayed runs give the same bits.

dh1 = ca*dz1 + (cb*h1 + cc) is staged as the kernel forms it: each fmaf in fp64 (the product of an
fp32 and a bf16 value is exact there) rounded once to fp32, then rounded to bf16.  The products
are long fp32 sums: |got - r| <= 2^-10 |r| + 2^-8 Q with Q = sqrt(sum of squared terms) (plus
one bf16 rounding of dx); a missing panel or unit changes a sum by a multiple of Q."""
import pytest
import torch

from expand_bwd_seq import ExpandBwd

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _inputs(M, Cin, Chid, residual, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)

    def bf(*shape, s=1.0):
        return (torch.randn(*shape, device=DEV, generator=g) * s).to(torch.bfloat16)

    def f32(n, s):
        return torch.randn(n, device=DEV, generator=g) * s

    return dict(dz1=bf(M, Chid), h1=bf(M, Chid), ca=f32(Chid, 1.0), cb=f32(Chid, 0.5),
                cc=f32(Chid, 0.1), w1=bf(Chid, Cin, s=0.2), x=bf(M, Cin),
                residual=bf(M, Cin) if residual else None)


def _dh1_ref(d):
    t = (d["cb"].double() * d["h1"].double() + d["cc"].double()).float()
    return (d["ca"].double() * d["dz1"].double() + t.double()).float().to(torch.bfloat16)


def _check(got, r, q, extra_rel, what):
    bound = 2.0 ** -10 * r.abs() + 2.0 ** -8 * q + extra_rel * r.abs()
    bad = (got.double() - r).abs() > bound
    assert not bad.any(), "%s: %d elements out of bound, first at %s" % (
        what, int(bad.sum()), tuple(bad.nonzero()[0].tolist()))


def _cases():
    out = []
    for cin in (16, 24, 32):
        for chid in (64, 96, 144, 192):
            out.append((cin, chid))
    return out


@pytest.mark.parametrize("cin,chid", _cases())
@pytest.mark.parametrize("residual", [False, True])
def test_expand_bwd_fp64(built_lib, cin, chid, residual):
    # at least two 128-pixel units per CTA and a partial last unit
    M = 2 * _sms() * 128 + 77
    d = _inputs(M, cin, chid, residual, seed=cin * 1000 + chid + residual)
    eb = ExpandBwd(d["dz1"], d["h1"], d["ca"], d["cb"], d["cc"], d["w1"], d["x"], d["residual"])
    eb.reset()
    eb.fused()
    torch.cuda.synchronize()
    dh = _dh1_ref(d).double()
    w = d["w1"].double()
    r_dx = dh @ w
    q_dx = ((dh * dh) @ (w * w)).sqrt()
    if residual:
        r_dx = r_dx + d["residual"].double()
    _check(eb.dx, r_dx, q_dx, 2.0 ** -8, "dx")
    xd = d["x"].double()
    r_dw = dh.t() @ xd
    q_dw = ((dh * dh).t() @ (xd * xd)).sqrt()
    _check(eb.dw1, r_dw, q_dw, 0.0, "dW1")


def _odd_slab_m(chid):
    """A pixel count whose split-K wgrad slabs are an odd number of 64-pixel k-blocks long (7), so
    that a slab ends in the middle of a 128-pixel unit, and whose last slab is partial."""
    want = 2 * _sms() // (1 if chid <= 128 else 2)
    return (want * 6 + 1) * 64 - 20


def _plan_info(eb):
    import ctypes as C
    info = eb.nat.ExpandBwdPlanInfo()
    assert eb.lib.yamb_expand_bwd_plan(C.byref(eb.args()), 0, C.byref(info)) == 0
    return info


@pytest.mark.parametrize("chid,cin", [(96, 16), (144, 24), (192, 32), (64, 8)])
@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("odd", [False, True])
def test_bitwise_equal_to_the_two_gemms(built_lib, chid, cin, residual, odd):
    """Same dh1 bits, same k order: the dgrad GEMM's dx and, slab by slab, the split-K wgrad's
    dW1 (added in the same slab order), bit for bit."""
    M = _odd_slab_m(chid) if odd else _sms() * 128 * 3 + 5
    d = _inputs(M, cin, chid, residual, seed=7 + chid)
    eb = ExpandBwd(d["dz1"], d["h1"], d["ca"], d["cb"], d["cc"], d["w1"], d["x"], d["residual"])
    eb.reset()
    eb.run("gemms")
    ref_dx, ref_dw = eb.dx.clone(), eb.dw1.clone()
    if odd:
        info = _plan_info(eb)
        assert info.slab_rows % 128 == 64 and M % info.slab_rows != 0
    init = torch.randn_like(ref_dw)
    eb.reset(init)
    eb.run("gemms")
    ref_acc = eb.dw1.clone()
    eb.reset()
    eb.run("fused")
    torch.cuda.synchronize()
    assert torch.equal(eb.dx, ref_dx)
    assert torch.equal(eb.dw1, ref_dw)
    eb.reset(init)
    eb.run("fused")
    torch.cuda.synchronize()
    assert torch.equal(eb.dw1, ref_acc)


def test_dw1_accumulates(built_lib):
    M = _sms() * 128 + 300
    d = _inputs(M, 32, 192, False, seed=11)
    eb = ExpandBwd(d["dz1"], d["h1"], d["ca"], d["cb"], d["cc"], d["w1"], d["x"])
    eb.reset()
    eb.fused()
    once = eb.dw1.clone()
    init = torch.randn_like(once)
    eb.reset(init)
    eb.fused()
    torch.cuda.synchronize()
    torch.testing.assert_close(eb.dw1, init + once, rtol=1e-5, atol=1e-5 * once.abs().max().item())
    eb.fused()
    torch.cuda.synchronize()
    torch.testing.assert_close(eb.dw1, init + 2 * once, rtol=1e-5,
                               atol=2e-5 * once.abs().max().item())


def test_repeatable_and_graph_replay(built_lib):
    M = 3 * _sms() * 128 + 19
    d = _inputs(M, 16, 96, True, seed=3)
    eb = ExpandBwd(d["dz1"], d["h1"], d["ca"], d["cb"], d["cc"], d["w1"], d["x"], d["residual"])
    outs = []
    for _ in range(2):
        eb.reset()
        eb.fused()
        torch.cuda.synchronize()
        outs.append((eb.dx.clone(), eb.dw1.clone()))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    eb.reset()
    torch.cuda.synchronize()
    with torch.cuda.graph(graph, stream=s):
        eb.fused()
    eb.reset()
    torch.cuda.synchronize()
    graph.replay()
    torch.cuda.synchronize()
    outs.append((eb.dx.clone(), eb.dw1.clone()))
    for dx, dw in outs[1:]:
        assert torch.equal(dx, outs[0][0])
        assert torch.equal(dw, outs[0][1])
