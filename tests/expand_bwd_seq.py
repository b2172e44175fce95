"""The expand-side backward of one block run two ways on the same inputs (GPU drivers and tests):

  gemms  dgrad GEMM dx = dh1 * W1 (+ dy) and split-K wgrad GEMM dW1 += dh1^T * x, each forming
         dh1 = ca1*dz1 + cb1*h1 + cc1 in its loaders (yamb_pointwise_gemm, two-source transform)
  fused  one yamb_expand_bwd launch that forms dh1 once and computes both products from it
"""
import ctypes as C

import torch


class ExpandBwd:
    def __init__(self, dz1, h1, ca, cb, cc, w1, x, residual=None):
        from yet_another_mobilenet_series_b200 import native as nat
        self.nat, self.lib = nat, nat.lib()
        self.M, self.Chid = dz1.shape
        self.Cin = x.shape[1]
        self.dz1, self.h1, self.ca, self.cb, self.cc = dz1, h1, ca, cb, cc
        self.w1, self.x, self.residual = w1, x, residual
        self.dx = torch.empty(self.M, self.Cin, device=dz1.device, dtype=torch.bfloat16)
        self.dw1 = torch.zeros(self.Chid, self.Cin, device=dz1.device, dtype=torch.float32)

    def reset(self, dw1=None):
        self.dx.fill_(float("nan"))
        if dw1 is None:
            self.dw1.zero_()
        else:
            self.dw1.copy_(dw1)

    def _check(self, rc):
        self.nat.check(rc)

    def dgrad(self):
        g = self.nat.Gemm()
        g.M, g.N, g.K = self.M, self.Cin, self.Chid
        g.A, g.lda = self.dz1.data_ptr(), self.Chid
        g.a_xform = 2
        g.a_scale, g.a_scale2, g.a_shift = self.ca.data_ptr(), self.cb.data_ptr(), self.cc.data_ptr()
        g.A2, g.lda2 = self.h1.data_ptr(), self.Chid
        g.B, g.ldb, g.b_mn_major = self.w1.data_ptr(), self.Cin, 1
        g.D, g.ldd = self.dx.data_ptr(), self.Cin
        if self.residual is not None:
            g.residual, g.ldr = self.residual.data_ptr(), self.Cin
        self._check(self.lib.yamb_pointwise_gemm(C.byref(g), self.nat.stream_handle()))

    def wgrad(self):
        g = self.nat.Gemm()
        g.M, g.N, g.K = self.Chid, self.Cin, self.M
        g.a_mn_major = g.b_mn_major = 1
        g.A, g.lda = self.dz1.data_ptr(), self.Chid
        g.a_xform = 2
        g.a_scale, g.a_scale2, g.a_shift = self.ca.data_ptr(), self.cb.data_ptr(), self.cc.data_ptr()
        g.A2, g.lda2 = self.h1.data_ptr(), self.Chid
        g.B, g.ldb = self.x.data_ptr(), self.Cin
        g.D, g.ldd = self.dw1.data_ptr(), self.Cin
        g.epi = 2
        self._check(self.lib.yamb_pointwise_gemm(C.byref(g), self.nat.stream_handle()))

    def args(self):
        a = self.nat.ExpandBwd()
        a.M, a.Cin, a.Chid = self.M, self.Cin, self.Chid
        a.dz1, a.h1 = self.dz1.data_ptr(), self.h1.data_ptr()
        a.ca, a.cb, a.cc = self.ca.data_ptr(), self.cb.data_ptr(), self.cc.data_ptr()
        a.W1, a.x = self.w1.data_ptr(), self.x.data_ptr()
        a.residual = None if self.residual is None else self.residual.data_ptr()
        a.dx, a.dW1 = self.dx.data_ptr(), self.dw1.data_ptr()
        return a

    def fused(self):
        self._check(self.lib.yamb_expand_bwd(C.byref(self.args()), self.nat.stream_handle()))

    def run(self, seq):
        if seq == "fused":
            self.fused()
        else:
            self.dgrad()
            self.wgrad()

    def nbytes(self, seq):
        """Algorithmic bytes of engine.py's launch tags."""
        M, Ch, Ci, r = self.M, self.Chid, self.Cin, self.residual is not None
        if seq == "fused":
            return 2 * M * (2 * Ch + Ci * (3 if r else 2))
        return 2 * M * (2 * Ch + Ci * (2 if r else 1)) + 2 * M * (2 * Ch + Ci)
