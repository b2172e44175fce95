// Eval-mode inverted-residual block in one launch, the hidden slices of every tile split over the
// CTAs of a thread-block cluster (small batches).  The kernel and its launch plan are in
// block_eval.cuh; a separate translation unit so that the two sets of instantiations compile in
// parallel.
#include "block_eval.cuh"

namespace yamb {

int block_eval_cluster_launch(const yamb_block_eval* a, int cluster, cudaStream_t st) {
  return block_eval_launch_impl<true>(a, st, false, cluster);
}

int block_eval_cluster_pool_launch(const yamb_block_eval* a, int cluster, cudaStream_t st) {
  return block_eval_launch_impl<true>(a, st, true, cluster);
}

}  // namespace yamb
