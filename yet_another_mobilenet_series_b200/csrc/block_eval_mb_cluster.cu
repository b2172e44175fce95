// Eval-mode multi-branch block (block_eval_mb.cu) in one launch, the 64-channel slices of the packed
// hidden dimension of every output tile split over the CTAs of a thread-block cluster (small
// batches).  Each slice runs the stencil of its own group whatever rank holds it, so the split is the
// single-branch one of block_eval.cuh (CLUSTER) over the packed tensors.  A separate translation unit
// so that its instantiations compile in parallel with the unsplit ones.
#include "block_eval_mb.cuh"

namespace yamb {

int block_eval_mb_cluster_launch(const yamb_block_eval_mb* m, bool pool, int cs, cudaStream_t st) {
  if (!m) return set_error(YAMB_EINVAL, "null args");
  if (cs != 2 && cs != 4 && cs != 8)
    return set_error(YAMB_EINVAL, "block_eval_mb: cluster size must be 2, 4 or 8 (got %d)", cs);
  int rc = block_eval_mb_check(m);
  if (rc) return rc;
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  const yamb_block_eval* a = &m->base;
  BlockEvalDev p;
  if ((rc = block_eval_setup(a, pool, cs, p))) return rc;
  block_eval_mb_groups(m, p);
  // the tile plan of block_eval_mb_launch
  const bool wide = p.Npad > 16 * kMaxProjChunks;
  auto tiles_of = [&](int toh, int tow, int ti) {
    return (long long)((p.Ho + toh - 1) / toh) * ((p.Wo + tow - 1) / tow) * ((a->N + ti - 1) / ti);
  };
  if (a->kernel == 5) {
    if (a->stride == 2) return launch_eval<EvGeomMB<5, 2, 6, 7, 1, 2>, true, true>(p, a, st);
    if (wide) return launch_eval<EvGeomMB<5, 1, 7, 7, 1, 4>, true, true>(p, a, st);
    if (tiles_of(7, 16, 1) <= tiles_of(7, 7, 2))
      return launch_eval<EvGeomMB<5, 1, 7, 16, 1, 4>, true, true>(p, a, st);
    return launch_eval<EvGeomMB<5, 1, 7, 7, 2, 4>, true, true>(p, a, st);
  }
  if (a->stride == 2) return launch_eval<EvGeomMB<7, 2, 4, 7, 1, 2>, true, true>(p, a, st);
  return launch_eval<EvGeomMB<7, 1, 7, 7, 1, 2>, true, true>(p, a, st);
}

}  // namespace yamb
