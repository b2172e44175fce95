// Depthwise k x k convolution: the 8- and 16-channel-tile instantiations (kernels: depthwise.cuh)
// for the narrow branches of searched networks (AtomNAS: apps/searched/models/atomnas_c.yml keeps
// branches of 1-23 channels; padded to multiples of 8 they are 8, 16 or 24 wide).  A separate
// translation unit so that the two sets of instantiations compile in parallel.
#include "depthwise.cuh"

namespace yamb {

int dw_fwd_dispatch_narrow(const DwFwdDev& p, int k, int s, int ct, int tw, size_t smem,
                           cudaStream_t st, int* grid) {
#define YAMB_FWD_CASE(KK, SS, CC, TT) \
  if (k == KK && s == SS && ct == CC && tw == TT) return grid ? grid_k("dw fwd launch", dw_fwd_kernel<KK, SS, CC, TT>, p, smem, p.num_tiles, grid) : launch_k(dw_fwd_kernel<KK, SS, CC, TT>, p, smem, p.num_tiles, st)
  YAMB_FWD_CASE(3, 1, 16, 1); YAMB_FWD_CASE(3, 1, 16, 2); YAMB_FWD_CASE(3, 2, 16, 1); YAMB_FWD_CASE(3, 2, 16, 2);
  YAMB_FWD_CASE(3, 1, 8, 1); YAMB_FWD_CASE(3, 1, 8, 2); YAMB_FWD_CASE(3, 2, 8, 1); YAMB_FWD_CASE(3, 2, 8, 2);
  YAMB_FWD_CASE(5, 1, 16, 1); YAMB_FWD_CASE(5, 1, 16, 2); YAMB_FWD_CASE(5, 2, 16, 1); YAMB_FWD_CASE(5, 2, 16, 2);
  YAMB_FWD_CASE(5, 1, 8, 1); YAMB_FWD_CASE(5, 1, 8, 2); YAMB_FWD_CASE(5, 2, 8, 1); YAMB_FWD_CASE(5, 2, 8, 2);
  YAMB_FWD_CASE(7, 1, 16, 1); YAMB_FWD_CASE(7, 2, 16, 1); YAMB_FWD_CASE(7, 1, 8, 1); YAMB_FWD_CASE(7, 2, 8, 1);
#undef YAMB_FWD_CASE
  return set_error(YAMB_ECUDA, "dw fwd launch: no kernel for k=%d stride=%d ct=%d tw=%d", k, s, ct, tw);
}

int dw_bwd_dispatch_narrow(const DwBwdDev& p, int k, int s, int ct, size_t smem, cudaStream_t st,
                           int* grid) {
  int rc;
  if (k == 3 && s == 1 && ct == 16) YAMB_DW_BWD(3, 1, 16, p, smem, p.num_tiles, st, grid);
  else if (k == 3 && s == 2 && ct == 16) YAMB_DW_BWD(3, 2, 16, p, smem, p.num_tiles, st, grid);
  else if (k == 3 && s == 1 && ct == 8) YAMB_DW_BWD(3, 1, 8, p, smem, p.num_tiles, st, grid);
  else if (k == 3 && s == 2 && ct == 8) YAMB_DW_BWD(3, 2, 8, p, smem, p.num_tiles, st, grid);
  else if (k == 5 && s == 1 && ct == 16) YAMB_DW_BWD(5, 1, 16, p, smem, p.num_tiles, st, grid);
  else if (k == 5 && s == 2 && ct == 16) YAMB_DW_BWD(5, 2, 16, p, smem, p.num_tiles, st, grid);
  else if (k == 5 && s == 1 && ct == 8) YAMB_DW_BWD(5, 1, 8, p, smem, p.num_tiles, st, grid);
  else if (k == 5 && s == 2 && ct == 8) YAMB_DW_BWD(5, 2, 8, p, smem, p.num_tiles, st, grid);
  else if (k == 7 && s == 1 && ct == 16) YAMB_DW_BWD(7, 1, 16, p, smem, p.num_tiles, st, grid);
  else if (k == 7 && s == 2 && ct == 16) YAMB_DW_BWD(7, 2, 16, p, smem, p.num_tiles, st, grid);
  else if (k == 7 && s == 1 && ct == 8) YAMB_DW_BWD(7, 1, 8, p, smem, p.num_tiles, st, grid);
  else if (k == 7 && s == 2 && ct == 8) YAMB_DW_BWD(7, 2, 8, p, smem, p.num_tiles, st, grid);
  else rc = set_error(YAMB_ECUDA, "dw bwd launch: no kernel for k=%d stride=%d ct=%d", k, s, ct);
  return rc;
}

}  // namespace yamb
