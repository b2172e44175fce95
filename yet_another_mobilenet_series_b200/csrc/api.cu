// C ABI entry points (include/yamb200.h) + host utilities.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>

#include <map>
#include <mutex>
#include <utility>

#include "host_util.h"

namespace yamb {

static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int max_ctas() {
  static int cached = 0;
  if (cached != 0) return cached;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return cached = -1; }
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
    cudaGetLastError();
    return cached = -1;
  }
  return cached = sms;
}

int smem_optin(const char* fn, const void* kern, size_t smem, int* per_sm, int block,
               bool max_carveout) {
  struct State {
    size_t static_smem;
    int optin;
    size_t raised;                          // the kernel's dynamic limit on this device, 0: default
    std::map<std::pair<int, size_t>, int> per_sm;   // (block, smem) -> resident CTAs per SM
  };
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, State> states;   // (kernel, device)
  auto fail = [fn](cudaError_t e) {
    cudaGetLastError();
    return set_error(YAMB_ECUDA, "%s: %s", fn, cudaGetErrorString(e));
  };
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return fail(e);
  std::lock_guard<std::mutex> lock(mu);
  auto it = states.find({kern, dev});
  if (it == states.end()) {
    State s{0, 0, 0, {}};
    cudaFuncAttributes fa;
    e = cudaFuncGetAttributes(&fa, kern);
    if (e == cudaSuccess)
      e = cudaDeviceGetAttribute(&s.optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (e == cudaSuccess && max_carveout)
      e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                               (int)cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return fail(e);
    s.static_smem = fa.sharedSizeBytes;
    it = states.emplace(std::make_pair(kern, dev), s).first;
  }
  State& s = it->second;
  const size_t total = s.static_smem + smem;
  if (total > (size_t)s.optin)
    return set_error(YAMB_EINVAL, "%s: needs %zu B of shared memory, the device allows %d B", fn,
                     total, s.optin);
  if (smem > s.raised && total > 48 * 1024) {
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail(e);
    s.raised = smem;
  }
  if (per_sm) {
    auto o = s.per_sm.find({block, smem});
    if (o == s.per_sm.end()) {
      int n = 0;
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, block, smem);
      if (e != cudaSuccess) return fail(e);
      o = s.per_sm.emplace(std::make_pair(block, smem), n).first;
    }
    *per_sm = o->second;
  }
  return 0;
}

PFN_encodeTiled get_encode_tiled() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) !=
          cudaSuccess ||
      qres != cudaDriverEntryPointSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return reinterpret_cast<PFN_encodeTiled>(fn);
}

}  // namespace yamb

extern "C" {

const char* yamb_last_error(void) { return yamb::g_err; }
int yamb_version(void) { return 103; }
int yamb_max_ctas(void) { int n = yamb::max_ctas(); return n > 0 ? 4 * n : n; }
int yamb_struct_size(int which) {
  switch (which) {
    case 0: return (int)sizeof(yamb_bn_fwd);
    case 1: return (int)sizeof(yamb_bn_bwd);
    case 2: return (int)sizeof(yamb_gemm);
    case 3: return (int)sizeof(yamb_dw_fwd);
    case 4: return (int)sizeof(yamb_dw_bwd);
    case 5: return (int)sizeof(yamb_bn_apply);
    case 6: return (int)sizeof(yamb_bn_reduce);
    case 7: return (int)sizeof(yamb_se_pool);
    case 8: return (int)sizeof(yamb_rmsprop);
    case 9: return (int)sizeof(yamb_se_bwd_reduce);
    case 10: return (int)sizeof(yamb_se_bwd_apply);
    case 11: return (int)sizeof(yamb_bn_stats);
    case 12: return (int)sizeof(yamb_bn_bwd_apply);
    case 13: return (int)sizeof(yamb_nl_gram);
    case 14: return (int)sizeof(yamb_nl_rowmat);
    case 15: return (int)sizeof(yamb_se_fc);
    case 16: return (int)sizeof(yamb_se_fc_grad);
    case 17: return (int)sizeof(yamb_softmax_ce);
    case 18: return (int)sizeof(yamb_softmax_ce_grad);
    case 19: return (int)sizeof(yamb_stem_conv);
    case 20: return (int)sizeof(yamb_bn_eval);
    case 21: return (int)sizeof(yamb_block_eval);
    case 22: return (int)sizeof(yamb_in_fwd);
    case 23: return (int)sizeof(yamb_in_bwd);
    case 24: return (int)sizeof(yamb_sgd);
    case 25: return (int)sizeof(yamb_stem_conv_eval);
    case 26: return (int)sizeof(yamb_head_pool_eval);
    case 27: return (int)sizeof(yamb_gemm_plan_info);
    case 28: return (int)sizeof(yamb_stem_conv_u8);
    case 29: return (int)sizeof(yamb_expand_bwd_args);
    case 30: return (int)sizeof(yamb_expand_bwd_plan_info);
    case 31: return (int)sizeof(yamb_head_pool_train);
    case 32: return (int)sizeof(yamb_head_pool_train_grad);
    case 33: return (int)sizeof(yamb_stem_conv_train);
    case 34: return (int)sizeof(yamb_stem_conv_train_grad);
    case 35: return (int)sizeof(yamb_block_eval_mb_pack_args);
    case 36: return (int)sizeof(yamb_block_eval_mb);
    case 37: return (int)sizeof(yamb_se_bwd_stats);
    case 38: return (int)sizeof(yamb_se_bn_bwd_finalize_args);
    case 39: return (int)sizeof(yamb_dw_bwd_se);
    case 40: return (int)sizeof(yamb_expand_dw_train);
    case 41: return (int)sizeof(yamb_dw_fwd_grouped);
    case 42: return (int)sizeof(yamb_dw_bwd_grouped);
    default: return -1;
  }
}

int yamb_pointwise_gemm(const yamb_gemm* args, yamb_stream_t stream) {
  return yamb::gemm_launch(args, reinterpret_cast<cudaStream_t>(stream));
}
int yamb_gemm_plan(const yamb_gemm* args, int32_t num_sms, yamb_gemm_plan_info* out) {
  return yamb::gemm_plan_query(args, num_sms, out);
}
int yamb_expand_bwd(const yamb_expand_bwd_args* args, yamb_stream_t stream) {
  return yamb::expand_bwd_launch(args, reinterpret_cast<cudaStream_t>(stream));
}
int yamb_expand_bwd_plan(const yamb_expand_bwd_args* args, int32_t num_sms, yamb_expand_bwd_plan_info* out) {
  return yamb::expand_bwd_plan_query(args, num_sms, out);
}


#define YAMB_ST(s) reinterpret_cast<cudaStream_t>(s)
int yamb_depthwise_fwd(const yamb_dw_fwd* a, yamb_stream_t s) { return yamb::dw_fwd_launch(a, YAMB_ST(s)); }
int yamb_depthwise_bwd(const yamb_dw_bwd* a, yamb_stream_t s) { return yamb::dw_bwd_launch(a, YAMB_ST(s)); }
int yamb_depthwise_fwd_grouped(const yamb_dw_fwd_grouped* a, yamb_stream_t s) {
  return yamb::dw_fwd_grouped_launch(a, YAMB_ST(s));
}
int yamb_depthwise_bwd_grouped(const yamb_dw_bwd_grouped* a, yamb_stream_t s) {
  return yamb::dw_bwd_grouped_launch(a, YAMB_ST(s));
}
int yamb_depthwise_grouped_grids(yamb_dw_fwd_grouped* f, yamb_dw_bwd_grouped* b) {
  return yamb::dw_grouped_grids(f, b);
}
int yamb_bn_apply_fwd(const yamb_bn_apply* a, yamb_stream_t s) { return yamb::bn_apply_launch(a, YAMB_ST(s)); }
int yamb_bn_reduce_bwd(const yamb_bn_reduce* a, yamb_stream_t s) { return yamb::bn_reduce_launch(a, YAMB_ST(s)); }
int yamb_bn_stats_fwd(const yamb_bn_stats* a, yamb_stream_t s) { return yamb::bn_stats_launch(a, YAMB_ST(s)); }
int yamb_bn_bwd_apply_bwd(const yamb_bn_bwd_apply* a, yamb_stream_t s) { return yamb::bn_bwd_apply_launch(a, YAMB_ST(s)); }
int yamb_se_pool_fwd(const yamb_se_pool* a, yamb_stream_t s) { return yamb::se_pool_launch(a, YAMB_ST(s)); }
int yamb_se_bwd_reduce_bwd(const yamb_se_bwd_reduce* a, yamb_stream_t s) { return yamb::se_bwd_reduce_launch(a, YAMB_ST(s)); }
int yamb_se_bwd_apply_bwd(const yamb_se_bwd_apply* a, yamb_stream_t s) { return yamb::se_bwd_apply_launch(a, YAMB_ST(s)); }
int yamb_se_bwd_stats_bwd(const yamb_se_bwd_stats* a, yamb_stream_t s) { return yamb::se_bwd_stats_launch(a, YAMB_ST(s)); }
int yamb_se_bn_bwd_finalize(const yamb_se_bn_bwd_finalize_args* a, yamb_stream_t s) { return yamb::se_bn_bwd_finalize_launch(a, YAMB_ST(s)); }
int yamb_depthwise_bwd_se(const yamb_dw_bwd_se* a, yamb_stream_t s) { return yamb::dw_bwd_se_launch(a, YAMB_ST(s)); }
int yamb_se_fc_fwd(const yamb_se_fc* a, yamb_stream_t s) { return yamb::se_fc_fwd_launch(a, YAMB_ST(s)); }
int yamb_se_fc_bwd(const yamb_se_fc_grad* a, yamb_stream_t s) { return yamb::se_fc_bwd_launch(a, YAMB_ST(s)); }
int yamb_softmax_ce_fwd(const yamb_softmax_ce* a, yamb_stream_t s) { return yamb::softmax_ce_fwd_launch(a, YAMB_ST(s)); }
int yamb_softmax_ce_bwd(const yamb_softmax_ce_grad* a, yamb_stream_t s) { return yamb::softmax_ce_bwd_launch(a, YAMB_ST(s)); }
int yamb_colsum_bf16(const void* X, int64_t M, int32_t C, int64_t ld, float* out, yamb_stream_t s) {
  return yamb::colsum_bf16_launch(X, M, C, ld, out, YAMB_ST(s));
}
int yamb_stem_conv_fwd(const yamb_stem_conv* a, yamb_stream_t s) { return yamb::stem_conv_fwd_launch(a, YAMB_ST(s)); }
int yamb_stem_conv_wgrad(const yamb_stem_conv* a, yamb_stream_t s) { return yamb::stem_conv_wgrad_launch(a, YAMB_ST(s)); }
int yamb_stem_conv_eval_fwd(const yamb_stem_conv_eval* a, yamb_stream_t s) { return yamb::stem_conv_eval_fwd_launch(a, YAMB_ST(s)); }
int yamb_stem_conv_u8_fwd(const yamb_stem_conv_u8* a, yamb_stream_t s) { return yamb::stem_conv_u8_fwd_launch(a, YAMB_ST(s)); }
int yamb_stem_conv_u8_wgrad(const yamb_stem_conv_u8* a, yamb_stream_t s) { return yamb::stem_conv_u8_wgrad_launch(a, YAMB_ST(s)); }
int yamb_stem_conv_u8_eval_fwd(const yamb_stem_conv_u8* a, yamb_stream_t s) { return yamb::stem_conv_u8_eval_fwd_launch(a, YAMB_ST(s)); }
int yamb_stem_conv_train_fwd(const yamb_stem_conv_train* a, yamb_stream_t s) { return yamb::stem_conv_train_fwd_launch(a, YAMB_ST(s)); }
int yamb_stem_conv_train_wgrad(const yamb_stem_conv_train_grad* a, yamb_stream_t s) { return yamb::stem_conv_train_wgrad_launch(a, YAMB_ST(s)); }
int yamb_head_pool_eval_fwd(const yamb_head_pool_eval* a, yamb_stream_t s) { return yamb::head_pool_eval_launch(a, YAMB_ST(s)); }
int yamb_head_pool_train_fwd(const yamb_head_pool_train* a, yamb_stream_t s) { return yamb::head_pool_train_fwd_launch(a, YAMB_ST(s)); }
int yamb_head_pool_train_bwd(const yamb_head_pool_train_grad* a, yamb_stream_t s) { return yamb::head_pool_train_bwd_launch(a, YAMB_ST(s)); }
int yamb_nl_gram_fwd(const yamb_nl_gram* a, yamb_stream_t s) { return yamb::nl_gram_launch(a, YAMB_ST(s)); }
int yamb_nl_rowmat_fwd(const yamb_nl_rowmat* a, yamb_stream_t s) { return yamb::nl_rowmat_launch(a, YAMB_ST(s)); }
int yamb_block_eval_fwd(const yamb_block_eval* a, yamb_stream_t s) { return yamb::block_eval_launch(a, YAMB_ST(s)); }
int yamb_block_eval_pool_fwd(const yamb_block_eval* a, yamb_stream_t s) { return yamb::block_eval_pool_launch(a, YAMB_ST(s)); }
int yamb_block_eval_cluster_fwd(const yamb_block_eval* a, int32_t cluster, yamb_stream_t s) {
  return yamb::block_eval_cluster_launch(a, cluster, YAMB_ST(s));
}
int yamb_block_eval_cluster_pool_fwd(const yamb_block_eval* a, int32_t cluster, yamb_stream_t s) {
  return yamb::block_eval_cluster_pool_launch(a, cluster, YAMB_ST(s));
}
int yamb_block_eval_mb_pack(const yamb_block_eval_mb_pack_args* a, yamb_stream_t s) {
  return yamb::block_eval_mb_pack_launch(a, YAMB_ST(s));
}
int yamb_block_eval_mb_fwd(const yamb_block_eval_mb* a, yamb_stream_t s) {
  return yamb::block_eval_mb_launch(a, false, YAMB_ST(s));
}
int yamb_block_eval_mb_pool_fwd(const yamb_block_eval_mb* a, yamb_stream_t s) {
  return yamb::block_eval_mb_launch(a, true, YAMB_ST(s));
}
int yamb_block_eval_mb_cluster_fwd(const yamb_block_eval_mb* a, int32_t cluster, yamb_stream_t s) {
  return yamb::block_eval_mb_cluster_launch(a, false, cluster, YAMB_ST(s));
}
int yamb_block_eval_mb_cluster_pool_fwd(const yamb_block_eval_mb* a, int32_t cluster, yamb_stream_t s) {
  return yamb::block_eval_mb_cluster_launch(a, true, cluster, YAMB_ST(s));
}
int yamb_expand_dw_train_fwd(const yamb_expand_dw_train* a, yamb_stream_t s) {
  return yamb::expand_dw_train_launch(a, YAMB_ST(s));
}
int yamb_instance_norm_fwd(const yamb_in_fwd* a, yamb_stream_t s) { return yamb::in_fwd_launch(a, YAMB_ST(s)); }
int yamb_instance_norm_bwd(const yamb_in_bwd* a, yamb_stream_t s) { return yamb::in_bwd_launch(a, YAMB_ST(s)); }
int yamb_rmsprop_step(const yamb_rmsprop* a, yamb_stream_t s) { return yamb::rmsprop_launch(a, YAMB_ST(s)); }
int yamb_sgd_step(const yamb_sgd* a, yamb_stream_t s) { return yamb::sgd_launch(a, YAMB_ST(s)); }
int yamb_ema_update(float* shadow, const float* x, int64_t n, const float* hyper, float m,
                    yamb_stream_t s) {
  return yamb::ema_launch(shadow, x, n, hyper, m, YAMB_ST(s));
}
int yamb_cast_bf16(const float* src, void* dst, int64_t n, yamb_stream_t s) {
  return yamb::cast_bf16_launch(src, dst, n, YAMB_ST(s));
}

}  // extern "C"
