// Depthwise backward of a Squeeze-and-Excitation block (yamb_depthwise_bwd_se): host side and the
// 32 / 64-channel-tile instantiations of dw_bwd_se_kernel (kernels: depthwise.cuh; 8 / 16-channel
// tiles: depthwise_se_narrow.cu).
#include "depthwise.cuh"

namespace yamb {

int dw_bwd_se_dispatch(const DwBwdSeDev& p, int k, int s, int ct, size_t smem, cudaStream_t st) {
  int rc;
  const long long nt = p.dw.num_tiles;
  if (k == 3 && s == 1 && ct == 64) YAMB_DW_BWD(3, 1, 64, p, smem, nt, st);
  else if (k == 3 && s == 2 && ct == 64) YAMB_DW_BWD(3, 2, 64, p, smem, nt, st);
  else if (k == 3 && s == 1 && ct == 32) YAMB_DW_BWD(3, 1, 32, p, smem, nt, st);
  else if (k == 3 && s == 2 && ct == 32) YAMB_DW_BWD(3, 2, 32, p, smem, nt, st);
  else if (k == 5 && s == 1 && ct == 64) YAMB_DW_BWD(5, 1, 64, p, smem, nt, st);
  else if (k == 5 && s == 2 && ct == 64) YAMB_DW_BWD(5, 2, 64, p, smem, nt, st);
  else if (k == 5 && s == 1 && ct == 32) YAMB_DW_BWD(5, 1, 32, p, smem, nt, st);
  else if (k == 5 && s == 2 && ct == 32) YAMB_DW_BWD(5, 2, 32, p, smem, nt, st);
  else if (k == 7 && s == 1 && ct == 64) YAMB_DW_BWD(7, 1, 64, p, smem, nt, st);
  else if (k == 7 && s == 2 && ct == 64) YAMB_DW_BWD(7, 2, 64, p, smem, nt, st);
  else if (k == 7 && s == 1 && ct == 32) YAMB_DW_BWD(7, 1, 32, p, smem, nt, st);
  else if (k == 7 && s == 2 && ct == 32) YAMB_DW_BWD(7, 2, 32, p, smem, nt, st);
  else rc = set_error(YAMB_ECUDA, "dw bwd se launch: no kernel for k=%d stride=%d ct=%d", k, s, ct);
  return rc;
}

int dw_bwd_se_launch(const yamb_dw_bwd_se* a, cudaStream_t st) {
  if (!a) return set_error(YAMB_EINVAL, "null args");
  // gate / dpool / scale / shift are read 8 channels (two float4) at a time from the slice's
  // first channel on
  if (!a->gate || !a->dpool || !a->scale || !a->shift)
    return set_error(YAMB_EINVAL, "depthwise bwd se: null pointer");
  if (((uintptr_t)a->gate | (uintptr_t)a->dpool | (uintptr_t)a->scale | (uintptr_t)a->shift) & 15)
    return set_error(YAMB_EINVAL, "depthwise bwd se: gate, dpool, scale and shift must be 16-byte aligned");
  if (a->ldg < a->dw.C || a->ldg % 4)
    return set_error(YAMB_EINVAL, "depthwise bwd se: ldg=%d needs >= C=%d and a multiple of 4",
                     a->ldg, a->dw.C);
  if (a->act < YAMB_ACT_NONE || a->act > YAMB_ACT_HSWISH)
    return set_error(YAMB_EINVAL, "depthwise bwd se: act=%d", a->act);
  DwBwdSeDev p;
  int ct;
  size_t smem;
  int rc = dw_bwd_setup(&a->dw, &p.dw, &ct, &smem);
  if (rc) return rc;
  p.se.gate = a->gate; p.se.dpool = a->dpool; p.se.ldg = a->ldg;
  p.se.scale = a->scale; p.se.shift = a->shift; p.se.act = a->act;
  if (ct <= 16) return dw_bwd_se_dispatch_narrow(p, a->dw.k, a->dw.stride, ct, smem, st);
  return dw_bwd_se_dispatch(p, a->dw.k, a->dw.stride, ct, smem, st);
}

}  // namespace yamb
