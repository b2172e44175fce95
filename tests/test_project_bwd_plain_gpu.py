"""The project-side backward forms dh3 = ca3*dy + cb3*h3 + cc3 once (yamb_bn_bwd_apply) and feeds
it to the dgrad and wgrad GEMMs as a plain operand.  Before, the GEMM loaders formed it per output
tile (two-source operand transform).  Both are the same fp32 expression rounded RN to bf16, so the
tensor-core operands, and everything computed from them, must agree bit for bit: dz2 (or d(a2*gate)
with an SE gate), the BN2-backward dgamma / dbeta / ca / cb / cc and dW3.

Shapes cover the register (Cout < 64) and TMA (Cout >= 64) transform paths of the old sequence,
Cout = 320, Chid not a multiple of 64, a last m-block of fewer than 128 rows, an SE gate and a
BN2 split into several modules (one dgrad launch per slice).  Sequences: tests/project_bwd_seq.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# name: (N, H*W, Cout, BN2 slice widths, activation code, SE gate)
CASES = {
    "cout24_reg": (8, 28 * 28, 24, [144], 2, False),
    "cout40_chid120_reg": (6, 14 * 14 + 3, 40, [120], 1, False),
    "cout64_tma": (8, 14 * 14, 64, [384], 2, False),
    "cout96_chid200_tma": (5, 7 * 7, 96, [200], 3, False),
    "cout320_tma": (16, 7 * 7, 320, [960], 2, False),
    "se_cout40_swish": (4, 14 * 14, 40, [240], 3, True),
    "se_cout112_hswish": (4, 7 * 7, 112, [336], 4, True),
    "multislice_cout32": (6, 14 * 14, 32, [48, 96, 48], 1, False),
    "multislice_cout80_swish": (4, 7 * 7 + 5, 80, [120, 240], 3, False),
}


def _inputs(N, HW, Cout, widths, act, se, seed):
    from project_bwd_seq import ProjectBwd
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev, bf = "cuda", torch.bfloat16
    M, Chid = N * HW, sum(widths)

    def rn(*s, sc=1.0, off=0.0):
        return torch.randn(*s, generator=g, device=dev) * sc + off

    def ru(*s, lo=0.5, hi=1.5):
        return torch.rand(*s, generator=g, device=dev) * (hi - lo) + lo

    dy = rn(M, Cout).to(bf)
    h3 = rn(M, Cout, sc=2.0, off=0.3).to(bf)
    h2 = rn(M, Chid, sc=1.5, off=0.2).to(bf)
    w3 = rn(Cout, Chid, sc=Chid ** -0.5).to(bf)
    # BN3-backward coefficients of the magnitudes a real batch gives: ca = gamma*invstd,
    # cb = -ca*invstd*mean(dy*xhat), cc = ca*(mean*invstd*mean(dy*xhat) - mean(dy))
    ca3, cb3, cc3 = ru(Cout), rn(Cout, sc=0.05), rn(Cout, sc=0.02)
    bn2 = {"scale": ru(Chid), "shift": rn(Chid, sc=0.3), "mean": rn(Chid, sc=0.2),
           "invstd": ru(Chid), "gamma": ru(Chid)}
    gate = torch.sigmoid(rn(N, Chid)) if se else None
    slices, c0 = [], 0
    for w in widths:
        slices.append((c0, w))
        c0 += w
    return ProjectBwd(dy, h3, h2, w3, ca3, cb3, cc3, bn2, act, HW,
                      slices=slices if len(slices) > 1 else None, gate=gate)


@pytest.mark.parametrize("name", list(CASES))
def test_plain_matches_loader_transform(built_lib, name):
    pb = _inputs(*CASES[name], seed=sorted(CASES).index(name) + 11)
    outs = {}
    for seq in ("xform", "plain", "xform"):
        pb.reset()
        pb.run(seq)
        torch.cuda.synchronize()
        o = pb.outputs()
        if seq in outs:                    # the old sequence repeated: its own bits again
            for k in o:
                assert torch.equal(o[k], outs[seq][k]), (name, "xform run-to-run", k)
        outs[seq] = o
    assert set(outs["plain"]) == set(outs["xform"])
    for k, want in outs["xform"].items():
        got = outs["plain"][k]
        assert torch.isfinite(got.float()).all(), (name, k)
        diff = int((got.view(torch.int16 if got.dtype == torch.bfloat16 else torch.int32)
                    != want.view(torch.int16 if want.dtype == torch.bfloat16 else torch.int32))
                   .sum())
        assert diff == 0, "%s: %s differs in %d of %d elements" % (name, k, diff, want.numel())
    # the outputs are not trivially equal: dz2 carries real values
    assert float(outs["plain"]["dz2"].float().abs().sum()) > 0
