// C ABI entry points (include/yamb200.h) + host utilities.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>

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
int yamb_version(void) { return 102; }
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
    default: return -1;
  }
}

int yamb_pointwise_gemm(const yamb_gemm* args, yamb_stream_t stream) {
  return yamb::gemm_launch(args, reinterpret_cast<cudaStream_t>(stream));
}


#define YAMB_ST(s) reinterpret_cast<cudaStream_t>(s)
int yamb_depthwise_fwd(const yamb_dw_fwd* a, yamb_stream_t s) { return yamb::dw_fwd_launch(a, YAMB_ST(s)); }
int yamb_depthwise_bwd(const yamb_dw_bwd* a, yamb_stream_t s) { return yamb::dw_bwd_launch(a, YAMB_ST(s)); }
int yamb_bn_apply_fwd(const yamb_bn_apply* a, yamb_stream_t s) { return yamb::bn_apply_launch(a, YAMB_ST(s)); }
int yamb_bn_reduce_bwd(const yamb_bn_reduce* a, yamb_stream_t s) { return yamb::bn_reduce_launch(a, YAMB_ST(s)); }
int yamb_bn_stats_fwd(const yamb_bn_stats* a, yamb_stream_t s) { return yamb::bn_stats_launch(a, YAMB_ST(s)); }
int yamb_bn_bwd_apply_bwd(const yamb_bn_bwd_apply* a, yamb_stream_t s) { return yamb::bn_bwd_apply_launch(a, YAMB_ST(s)); }
int yamb_se_pool_fwd(const yamb_se_pool* a, yamb_stream_t s) { return yamb::se_pool_launch(a, YAMB_ST(s)); }
int yamb_se_bwd_reduce_bwd(const yamb_se_bwd_reduce* a, yamb_stream_t s) { return yamb::se_bwd_reduce_launch(a, YAMB_ST(s)); }
int yamb_se_bwd_apply_bwd(const yamb_se_bwd_apply* a, yamb_stream_t s) { return yamb::se_bwd_apply_launch(a, YAMB_ST(s)); }
int yamb_se_fc_fwd(const yamb_se_fc* a, yamb_stream_t s) { return yamb::se_fc_fwd_launch(a, YAMB_ST(s)); }
int yamb_se_fc_bwd(const yamb_se_fc_grad* a, yamb_stream_t s) { return yamb::se_fc_bwd_launch(a, YAMB_ST(s)); }
int yamb_softmax_ce_fwd(const yamb_softmax_ce* a, yamb_stream_t s) { return yamb::softmax_ce_fwd_launch(a, YAMB_ST(s)); }
int yamb_softmax_ce_bwd(const yamb_softmax_ce_grad* a, yamb_stream_t s) { return yamb::softmax_ce_bwd_launch(a, YAMB_ST(s)); }
int yamb_colsum_bf16(const void* X, int64_t M, int32_t C, int64_t ld, float* out, yamb_stream_t s) {
  return yamb::colsum_bf16_launch(X, M, C, ld, out, YAMB_ST(s));
}
int yamb_stem_conv_fwd(const yamb_stem_conv* a, yamb_stream_t s) { return yamb::stem_conv_fwd_launch(a, YAMB_ST(s)); }
int yamb_stem_conv_wgrad(const yamb_stem_conv* a, yamb_stream_t s) { return yamb::stem_conv_wgrad_launch(a, YAMB_ST(s)); }
int yamb_nl_gram_fwd(const yamb_nl_gram* a, yamb_stream_t s) { return yamb::nl_gram_launch(a, YAMB_ST(s)); }
int yamb_nl_rowmat_fwd(const yamb_nl_rowmat* a, yamb_stream_t s) { return yamb::nl_rowmat_launch(a, YAMB_ST(s)); }
int yamb_block_eval_fwd(const yamb_block_eval* a, yamb_stream_t s) { return yamb::block_eval_launch(a, YAMB_ST(s)); }
int yamb_block_eval_pool_fwd(const yamb_block_eval* a, yamb_stream_t s) { return yamb::block_eval_pool_launch(a, YAMB_ST(s)); }
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
