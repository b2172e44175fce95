// Depthwise backward of a Squeeze-and-Excitation block: the 8- and 16-channel-tile instantiations
// of dw_bwd_se_kernel (kernels: depthwise.cuh), for the narrow branches of searched networks with
// SE (AtomNAS-A+/B+/C+).  A separate translation unit, compiled in parallel with depthwise_se.cu.
#include "depthwise.cuh"

namespace yamb {

int dw_bwd_se_dispatch_narrow(const DwBwdSeDev& p, int k, int s, int ct, size_t smem,
                              cudaStream_t st) {
  int rc;
  const long long nt = p.dw.num_tiles;
  if (k == 3 && s == 1 && ct == 16) YAMB_DW_BWD(3, 1, 16, p, smem, nt, st);
  else if (k == 3 && s == 2 && ct == 16) YAMB_DW_BWD(3, 2, 16, p, smem, nt, st);
  else if (k == 3 && s == 1 && ct == 8) YAMB_DW_BWD(3, 1, 8, p, smem, nt, st);
  else if (k == 3 && s == 2 && ct == 8) YAMB_DW_BWD(3, 2, 8, p, smem, nt, st);
  else if (k == 5 && s == 1 && ct == 16) YAMB_DW_BWD(5, 1, 16, p, smem, nt, st);
  else if (k == 5 && s == 2 && ct == 16) YAMB_DW_BWD(5, 2, 16, p, smem, nt, st);
  else if (k == 5 && s == 1 && ct == 8) YAMB_DW_BWD(5, 1, 8, p, smem, nt, st);
  else if (k == 5 && s == 2 && ct == 8) YAMB_DW_BWD(5, 2, 8, p, smem, nt, st);
  else if (k == 7 && s == 1 && ct == 16) YAMB_DW_BWD(7, 1, 16, p, smem, nt, st);
  else if (k == 7 && s == 2 && ct == 16) YAMB_DW_BWD(7, 2, 16, p, smem, nt, st);
  else if (k == 7 && s == 1 && ct == 8) YAMB_DW_BWD(7, 1, 8, p, smem, nt, st);
  else if (k == 7 && s == 2 && ct == 8) YAMB_DW_BWD(7, 2, 8, p, smem, nt, st);
  else rc = set_error(YAMB_ECUDA, "dw bwd se launch: no kernel for k=%d stride=%d ct=%d", k, s, ct);
  return rc;
}

}  // namespace yamb
