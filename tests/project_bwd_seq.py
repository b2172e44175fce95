"""The project-side backward of an inverted-residual block (project dgrad + BN2-backward statistics,
project wgrad) as two sequences of C-ABI launches, for comparing them bit for bit and timing them:

  "xform": the GEMM loaders form A = dh3 = ca3*dy + cb3*h3 + cc3 from dy and h3 (two-source
           operand transform), once per output tile, in both the dgrad and the wgrad;
  "plain": yamb_bn_bwd_apply forms dh3 once, both GEMMs read it as a plain operand (what
           engine.BlockPlan.backward runs).

The inputs are given as tensors, so the caller chooses random or recorded activations.  Used by
tests/test_project_bwd_plain_gpu.py and tests/gpu_project_bwd_bench.py."""
import ctypes as C

import torch

from yet_another_mobilenet_series_b200 import engine
from yet_another_mobilenet_series_b200 import native as nat


class ProjectBwd:
    """dy, h3: [M, Cout] bf16; h2: [M, Chid] bf16; w3: [Cout, Chid] bf16; ca3/cb3/cc3: [Cout] fp32;
    bn2: dict of [Chid] fp32 tensors scale, shift, mean, invstd, gamma; slices: BN2 module slices
    [(c0, width)] (one per module; the dgrad runs one launch per slice when there are several);
    gate: [N, Chid] fp32 SE gate or None (then the dgrad writes d(a2*gate), epilogue 0)."""

    def __init__(self, dy, h3, h2, w3, ca3, cb3, cc3, bn2, act, hw, slices=None, gate=None):
        self.dy, self.h3, self.h2, self.w3 = dy, h3, h2, w3
        self.ca3, self.cb3, self.cc3 = ca3, cb3, cc3
        self.bn2, self.act, self.hw, self.gate = bn2, act, hw, gate
        self.M, self.Cout = h3.shape
        self.Chid = h2.shape[1]
        self.slices = slices or [(0, self.Chid)]
        dev = h3.device
        f32 = dict(device=dev, dtype=torch.float32)
        self.dh3 = torch.empty_like(h3)
        self.dz2 = torch.empty_like(h2)
        self.dw3 = torch.zeros(self.Cout, self.Chid, **f32)
        self.co2 = {k: torch.zeros(self.Chid, **f32) for k in ("dgamma", "dbeta", "ca", "cb", "cc")}
        self._keep = []

    # -- one launch each ---------------------------------------------------------------------
    def apply(self):
        a = nat.BnBwdApply()
        a.M, a.C, a.lddy, a.ldh, a.lddh = self.M, self.Cout, self.Cout, self.Cout, self.Cout
        a.dy, a.h = self.dy.data_ptr(), self.h3.data_ptr()
        a.ca, a.cb, a.cc = self.ca3.data_ptr(), self.cb3.data_ptr(), self.cc3.data_ptr()
        a.dh = self.dh3.data_ptr()
        nat.check(nat.lib().yamb_bn_bwd_apply_bwd(C.byref(a), nat.stream_handle()))

    def _xform_a(self, g):
        g.a_xform = 2
        g.a_scale, g.a_scale2, g.a_shift = self.ca3.data_ptr(), self.cb3.data_ptr(), \
            self.cc3.data_ptr()
        g.A2, g.lda2 = self.h3.data_ptr(), self.Cout

    def _bn2_bwd(self, c0, cb):
        s = nat.BnBwd()
        ws = engine.Workspace.get(self.h2.device)
        s.partials, s.counter = ws.partials.data_ptr(), ws.counter.data_ptr()
        s.gamma = self.bn2["gamma"].data_ptr() + 4 * c0
        s.mean = self.bn2["mean"].data_ptr() + 4 * c0
        s.invstd = self.bn2["invstd"].data_ptr() + 4 * c0
        s.dgamma = self.co2["dgamma"].data_ptr() + 4 * c0
        s.dbeta = self.co2["dbeta"].data_ptr() + 4 * c0
        s.ca, s.cb, s.cc = (self.co2[k].data_ptr() + 4 * c0 for k in ("ca", "cb", "cc"))
        s.count = self.M
        s.use_batch_stats = 1
        self._keep.append(s)
        return s

    def dgrad(self, seq):
        g = nat.Gemm()
        g.M, g.N, g.K = self.M, self.Chid, self.Cout
        if seq == "xform":
            g.A, g.lda = self.dy.data_ptr(), self.Cout
            self._xform_a(g)
        else:
            g.A, g.lda = self.dh3.data_ptr(), self.Cout
        g.B, g.ldb, g.b_mn_major = self.w3.data_ptr(), self.Chid, 1
        g.D, g.ldd = self.dz2.data_ptr(), self.Chid
        lib = nat.lib()
        if self.gate is not None:
            nat.check(lib.yamb_pointwise_gemm(C.byref(g), nat.stream_handle()))
            return
        g.epi = 1
        g.H, g.ldh = self.h2.data_ptr(), self.Chid
        g.h_scale, g.h_shift, g.h_act = self.bn2["scale"].data_ptr(), \
            self.bn2["shift"].data_ptr(), self.act
        for c0, cb in self.slices:
            gs = nat.Gemm()
            C.memmove(C.byref(gs), C.byref(g), C.sizeof(nat.Gemm))
            gs.N = cb
            gs.B, gs.D, gs.H = g.B + 2 * c0, g.D + 2 * c0, g.H + 2 * c0
            gs.h_scale, gs.h_shift = g.h_scale + 4 * c0, g.h_shift + 4 * c0
            gs.bn_bwd = C.pointer(self._bn2_bwd(c0, cb))
            nat.check(lib.yamb_pointwise_gemm(C.byref(gs), nat.stream_handle()))

    def wgrad(self, seq):
        g = nat.Gemm()
        g.M, g.N, g.K = self.Cout, self.Chid, self.M
        g.a_mn_major = g.b_mn_major = 1
        if seq == "xform":
            g.A, g.lda = self.dy.data_ptr(), self.Cout
            self._xform_a(g)
        else:
            g.A, g.lda = self.dh3.data_ptr(), self.Cout
        g.B, g.ldb = self.h2.data_ptr(), self.Chid
        g.b_xform, g.b_act = 1, self.act
        g.b_scale, g.b_shift = self.bn2["scale"].data_ptr(), self.bn2["shift"].data_ptr()
        if self.gate is not None:
            g.b_gate, g.gate_rows_per_sample = self.gate.data_ptr(), self.hw
        g.D, g.ldd = self.dw3.data_ptr(), self.Chid
        g.epi = 2
        nat.check(nat.lib().yamb_pointwise_gemm(C.byref(g), nat.stream_handle()))

    # -- whole sequences -------------------------------------------------------------------------
    def reset(self):
        """Zero the accumulated outputs (dW3, BN2 dgamma / dbeta are accumulated with +=)."""
        self.dw3.zero_()
        for t in self.co2.values():
            t.zero_()
        self._keep = []

    def run(self, seq):
        if seq == "plain":
            self.apply()
        self.dgrad(seq)
        self.wgrad(seq)

    def outputs(self):
        """Copies of what the sequence computed (BN2 statistics only without an SE gate)."""
        out = {"dz2": self.dz2.clone(), "dW3": self.dw3.clone()}
        if self.gate is None:
            out.update({"bn2_" + k: t.clone() for k, t in self.co2.items()})
        return out
