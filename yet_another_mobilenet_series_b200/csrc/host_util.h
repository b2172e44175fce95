// Host-side helpers shared by the launchers: error reporting, device queries, driver entry points.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "../../include/yamb200.h"

namespace yamb {

int set_error(int code, const char* fmt, ...);
int max_ctas();  // SM count of the current device, <= 0 without a device

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_tiled();

int gemm_launch(const yamb_gemm* a, cudaStream_t stream);
int dw_fwd_launch(const yamb_dw_fwd* a, cudaStream_t stream);
int dw_bwd_launch(const yamb_dw_bwd* a, cudaStream_t stream);
int bn_apply_launch(const yamb_bn_apply* a, cudaStream_t stream);
int bn_reduce_launch(const yamb_bn_reduce* a, cudaStream_t stream);
int bn_stats_launch(const yamb_bn_stats* a, cudaStream_t stream);
int bn_bwd_apply_launch(const yamb_bn_bwd_apply* a, cudaStream_t stream);
int se_pool_launch(const yamb_se_pool* a, cudaStream_t stream);
int se_bwd_reduce_launch(const yamb_se_bwd_reduce* a, cudaStream_t stream);
int se_bwd_apply_launch(const yamb_se_bwd_apply* a, cudaStream_t stream);
int se_fc_fwd_launch(const yamb_se_fc* a, cudaStream_t stream);
int se_fc_bwd_launch(const yamb_se_fc_grad* a, cudaStream_t stream);
int softmax_ce_fwd_launch(const yamb_softmax_ce* a, cudaStream_t stream);
int softmax_ce_bwd_launch(const yamb_softmax_ce_grad* a, cudaStream_t stream);
int colsum_bf16_launch(const void* X, long long M, int C, long long ld, float* out,
                       cudaStream_t stream);
int stem_conv_fwd_launch(const yamb_stem_conv* a, cudaStream_t stream);
int stem_conv_wgrad_launch(const yamb_stem_conv* a, cudaStream_t stream);
int nl_gram_launch(const yamb_nl_gram* a, cudaStream_t stream);
int nl_rowmat_launch(const yamb_nl_rowmat* a, cudaStream_t stream);
int block_eval_launch(const yamb_block_eval* a, cudaStream_t stream);
int block_eval_pool_launch(const yamb_block_eval* a, cudaStream_t stream);
int in_fwd_launch(const yamb_in_fwd* a, cudaStream_t stream);
int in_bwd_launch(const yamb_in_bwd* a, cudaStream_t stream);
int rmsprop_launch(const yamb_rmsprop* a, cudaStream_t stream);
int sgd_launch(const yamb_sgd* a, cudaStream_t stream);
int ema_launch(float* shadow, const float* x, long long n, const float* hyper, float m,
               cudaStream_t stream);
int cast_bf16_launch(const float* src, void* dst, long long n, cudaStream_t stream);

// deterministic reductions (det_reduce.cu): a stream-ordered scratch per launch; det_reduce_launch
// adds its nslab slabs of n floats in slab order into out (add) or stores their sum (!add), and
// releases the scratch on the same stream
int det_alloc(size_t bytes, cudaStream_t stream, float** out);
int det_free(float* part, cudaStream_t stream);
int det_reduce_launch(float* part, int nslab, long long n, float* out, cudaStream_t stream,
                      bool add = true);

}  // namespace yamb
