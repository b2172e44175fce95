// Eval-mode inverted-residual block in one launch: the unsplit kernels (one CTA per output tile at
// a time).  The kernel and its launch plan are in block_eval.cuh.
#include "block_eval.cuh"

namespace yamb {

int block_eval_launch(const yamb_block_eval* a, cudaStream_t st) {
  return block_eval_launch_impl<false>(a, st, false, 1);
}

int block_eval_pool_launch(const yamb_block_eval* a, cudaStream_t st) {
  return block_eval_launch_impl<false>(a, st, true, 1);
}

}  // namespace yamb
