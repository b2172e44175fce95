// Host-side helpers shared by the launchers: error reporting, device queries, driver entry points.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "../../include/yamb200.h"

namespace yamb {

int set_error(int code, const char* fmt, ...);
int max_ctas();  // SM count of the current device, <= 0 without a device

// Dynamic shared memory for a launch of `kern` with `smem` bytes on the current device.  Refuses
// (YAMB_EINVAL, "`fn`: ... shared memory ...") when the kernel's static shared memory plus `smem`
// exceeds the device's opt-in maximum; past the 48 KiB default it raises the kernel's limit on this
// device, which is never lowered.  With `per_sm` it also returns the CTAs of `block` threads that
// are resident per SM at `smem`.  `max_carveout` asks for the largest shared-memory carveout (it
// shrinks the L1).  The state is per (kernel, device), under one lock: forward and backward
// launch from different host threads.  0 or a YAMB_* code with the message set.
int smem_optin(const char* fn, const void* kern, size_t smem, int* per_sm = nullptr,
               int block = 256, bool max_carveout = false);

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_tiled();

int gemm_launch(const yamb_gemm* a, cudaStream_t stream);
int gemm_plan_query(const yamb_gemm* a, int num_sms, yamb_gemm_plan_info* out);
int expand_bwd_launch(const yamb_expand_bwd_args* a, cudaStream_t stream);
int expand_bwd_plan_query(const yamb_expand_bwd_args* a, int num_sms, yamb_expand_bwd_plan_info* out);
int dw_fwd_launch(const yamb_dw_fwd* a, cudaStream_t stream);
int dw_bwd_launch(const yamb_dw_bwd* a, cudaStream_t stream);
int dw_fwd_grouped_launch(const yamb_dw_fwd_grouped* a, cudaStream_t stream);
int dw_bwd_grouped_launch(const yamb_dw_bwd_grouped* a, cudaStream_t stream);
int dw_grouped_grids(yamb_dw_fwd_grouped* fwd, yamb_dw_bwd_grouped* bwd);
int bn_apply_launch(const yamb_bn_apply* a, cudaStream_t stream);
int bn_reduce_launch(const yamb_bn_reduce* a, cudaStream_t stream);
int bn_stats_launch(const yamb_bn_stats* a, cudaStream_t stream);
int bn_bwd_apply_launch(const yamb_bn_bwd_apply* a, cudaStream_t stream);
int se_pool_launch(const yamb_se_pool* a, cudaStream_t stream);
int se_bwd_reduce_launch(const yamb_se_bwd_reduce* a, cudaStream_t stream);
int se_bwd_apply_launch(const yamb_se_bwd_apply* a, cudaStream_t stream);
int se_bwd_stats_launch(const yamb_se_bwd_stats* a, cudaStream_t stream);
int se_bn_bwd_finalize_launch(const yamb_se_bn_bwd_finalize_args* a, cudaStream_t stream);
int dw_bwd_se_launch(const yamb_dw_bwd_se* a, cudaStream_t stream);
int se_fc_fwd_launch(const yamb_se_fc* a, cudaStream_t stream);
int se_fc_bwd_launch(const yamb_se_fc_grad* a, cudaStream_t stream);
int softmax_ce_fwd_launch(const yamb_softmax_ce* a, cudaStream_t stream);
int softmax_ce_bwd_launch(const yamb_softmax_ce_grad* a, cudaStream_t stream);
int colsum_bf16_launch(const void* X, long long M, int C, long long ld, float* out,
                       cudaStream_t stream);
int stem_conv_fwd_launch(const yamb_stem_conv* a, cudaStream_t stream);
int stem_conv_wgrad_launch(const yamb_stem_conv* a, cudaStream_t stream);
int stem_conv_eval_fwd_launch(const yamb_stem_conv_eval* a, cudaStream_t stream);
int stem_conv_u8_fwd_launch(const yamb_stem_conv_u8* a, cudaStream_t stream);
int stem_conv_u8_wgrad_launch(const yamb_stem_conv_u8* a, cudaStream_t stream);
int stem_conv_u8_eval_fwd_launch(const yamb_stem_conv_u8* a, cudaStream_t stream);
int stem_conv_train_fwd_launch(const yamb_stem_conv_train* a, cudaStream_t stream);
int stem_conv_train_wgrad_launch(const yamb_stem_conv_train_grad* a, cudaStream_t stream);
int head_pool_eval_launch(const yamb_head_pool_eval* a, cudaStream_t stream);
int head_pool_train_fwd_launch(const yamb_head_pool_train* a, cudaStream_t stream);
int head_pool_train_bwd_launch(const yamb_head_pool_train_grad* a, cudaStream_t stream);
int nl_gram_launch(const yamb_nl_gram* a, cudaStream_t stream);
int nl_rowmat_launch(const yamb_nl_rowmat* a, cudaStream_t stream);
int block_eval_launch(const yamb_block_eval* a, cudaStream_t stream);
int block_eval_pool_launch(const yamb_block_eval* a, cudaStream_t stream);
int block_eval_cluster_launch(const yamb_block_eval* a, int cluster, cudaStream_t stream);
int block_eval_cluster_pool_launch(const yamb_block_eval* a, int cluster, cudaStream_t stream);
int block_eval_mb_pack_launch(const yamb_block_eval_mb_pack_args* a, cudaStream_t stream);
int block_eval_mb_launch(const yamb_block_eval_mb* a, bool pool, cudaStream_t stream);
int block_eval_mb_cluster_launch(const yamb_block_eval_mb* a, bool pool, int cluster, cudaStream_t stream);
int expand_dw_train_launch(const yamb_expand_dw_train* a, cudaStream_t stream);
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
