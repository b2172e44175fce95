// Label-smoothed softmax cross entropy + top-k correctness on bf16 logits, sm_90a.
//
// Replaces, behind yamb_softmax_ce_fwd / yamb_softmax_ce_bwd (include/yamb200.h), the ~20 ATen
// launches of the reference's loss path per step:
//   CrossEntropyLabelSmooth(reduction='none')   utils/optim.py:150-158
//     loss[n] = sum_c -t[n][c] * log_softmax(logits)[n][c],  t = (1-eps)*onehot + eps/C
//   the top-k bookkeeping of forward_loss        common.py:73-79  (k = 1, 5: `correct_k`)
// and their backward.  One warp per sample; the row stays in registers (C <= 4096).
//   forward : loss[n], correct1[n], correct5[n], G[n][c] = softmax[n][c] - t[n][c]  (bf16)
//   backward: dlogits[n][c] = G[n][c] * dloss[n]  (bf16)  and  dbias[c] += sum_n dlogits[n][c]
// No host synchronisation anywhere (the reference's forward_loss forces two per step).
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "host_util.h"
#include "prims.cuh"

namespace yamb {

constexpr int kCeMaxPerLane = 128;   // C <= 32 * 128

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_add(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(256) softmax_ce_fwd_kernel(const __grid_constant__ yamb_softmax_ce a) {
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (n >= a.N) return;
  const __nv_bfloat16* row = reinterpret_cast<const __nv_bfloat16*>(a.logits) + (size_t)n * a.ld;
  const long long tgt = a.target[n];
  // pass 1: max, target logit
  float mx = -3.0e38f;
  for (int c = lane; c < a.C; c += 32) mx = fmaxf(mx, __bfloat162float(row[c]));
  mx = warp_max(mx);
  const float tv = __bfloat162float(row[tgt]);
  // pass 2: sum exp, sum of logits, rank of the target (ties resolved like torch.topk: lower
  // index first)
  float se = 0.f, sl = 0.f;
  int above = 0;
  for (int c = lane; c < a.C; c += 32) {
    const float v = __bfloat162float(row[c]);
    se += __expf(v - mx);
    sl += v;
    above += (v > tv || (v == tv && c < tgt)) ? 1 : 0;
  }
  se = warp_add(se);
  sl = warp_add(sl);
  above = (int)warp_add((float)above);
  const float lse = mx + __logf(se);
  // loss = -(1-eps)*logp[t] - eps/C * sum_c logp[c]
  const float eps = a.smoothing;
  const float logp_t = tv - lse;
  const float sum_logp = sl - (float)a.C * lse;
  if (lane == 0) {
    a.loss[n] = -(1.f - eps) * logp_t - (eps / (float)a.C) * sum_logp;
    if (a.correct1) a.correct1[n] = above < 1 ? 1.f : 0.f;
    if (a.correct5) a.correct5[n] = above < 5 ? 1.f : 0.f;
  }
  if (a.G) {
    __nv_bfloat16* g = reinterpret_cast<__nv_bfloat16*>(a.G) + (size_t)n * a.ldg;
    const float u = eps / (float)a.C;
    for (int c = lane; c < a.C; c += 32) {
      const float p = __expf(__bfloat162float(row[c]) - lse);
      g[c] = __float2bfloat16_rn(p - u - (c == tgt ? (1.f - eps) : 0.f));
    }
  }
}

// dlogits = G * dloss[n]; dbias[c] += column sums.  grid-stride over rows, thread = column pair
__global__ void __launch_bounds__(256) softmax_ce_bwd_kernel(const __grid_constant__ yamb_softmax_ce_grad a,
                                                                      float* part) {
  const int CP = a.C / 2;
  for (int cp = threadIdx.x; cp < CP; cp += 256) {
    float b0 = 0.f, b1 = 0.f;
    for (int n = blockIdx.x; n < a.N; n += gridDim.x) {
      const float s = a.dloss[n];
      const uint32_t gv = reinterpret_cast<const uint32_t*>(
          reinterpret_cast<const __nv_bfloat16*>(a.G) + (size_t)n * a.ldg)[cp];
      const uint32_t o = pack_bf16(bf16lo(gv) * s, bf16hi(gv) * s);
      reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(a.dlogits) + (size_t)n * a.ldd)[cp] = o;
      b0 += bf16lo(o);
      b1 += bf16hi(o);
    }
    if (part) {   // per-CTA column sums, added in CTA order by det_reduce_launch
      part[(size_t)blockIdx.x * a.C + 2 * cp] = b0;
      part[(size_t)blockIdx.x * a.C + 2 * cp + 1] = b1;
    }
  }
}

// out[c] += sum_rows X[row][c]   (classifier bias gradient: column sums of dlogits)
__global__ void __launch_bounds__(256) colsum_bf16_kernel(const __nv_bfloat16* X, long long M, int C,
                                                          long long ld, float* part) {
  const int CP = C / 2;
  for (int cp = blockIdx.x * 256 + threadIdx.x; cp < CP; cp += gridDim.x * 256) {
    float b0 = 0.f, b1 = 0.f;
    for (long long r = blockIdx.y; r < M; r += gridDim.y) {
      const uint32_t v = reinterpret_cast<const uint32_t*>(X + r * ld)[cp];
      b0 += bf16lo(v);
      b1 += bf16hi(v);
    }
    part[(size_t)blockIdx.y * C + 2 * cp] = b0;     // row-slab sums, added in slab order
    part[(size_t)blockIdx.y * C + 2 * cp + 1] = b1;
  }
}

int colsum_bf16_launch(const void* X, long long M, int C, long long ld, float* out, cudaStream_t st) {
  if (!X || !out || M <= 0 || C <= 0 || (C % 2) || (ld % 2))
    return set_error(YAMB_EINVAL, "colsum args (C and ld must be even)");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  dim3 grid((C / 2 + 255) / 256, (unsigned)(M < 32 ? M : 32));
  float* part = nullptr;
  int rc = det_alloc((size_t)grid.y * C * sizeof(float), st, &part);
  if (rc) return rc;
  colsum_bf16_kernel<<<grid, 256, 0, st>>>((const __nv_bfloat16*)X, M, C, ld, part);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    det_free(part, st);
    return set_error(YAMB_ECUDA, "colsum: %s", cudaGetErrorString(e));
  }
  return det_reduce_launch(part, (int)grid.y, C, out, st);
}

int softmax_ce_fwd_launch(const yamb_softmax_ce* a, cudaStream_t st) {
  if (!a || a->N <= 0 || a->C <= 0 || a->C > 32 * kCeMaxPerLane || !a->logits || !a->target || !a->loss)
    return set_error(YAMB_EINVAL, "softmax_ce args");
  if (a->ld < a->C || (a->G && a->ldg < a->C)) return set_error(YAMB_EINVAL, "softmax_ce pitch");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  softmax_ce_fwd_kernel<<<(a->N + 7) / 8, 256, 0, st>>>(*a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "softmax_ce fwd: %s", cudaGetErrorString(e));
  return 0;
}

int softmax_ce_bwd_launch(const yamb_softmax_ce_grad* a, cudaStream_t st) {
  if (!a || a->N <= 0 || a->C <= 0 || (a->C % 2) || (a->ldg % 2) || (a->ldd % 2) || !a->G ||
      !a->dloss || !a->dlogits)
    return set_error(YAMB_EINVAL, "softmax_ce bwd args (C and pitches must be even)");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  int grid = a->N < 2 * max_ctas() ? a->N : 2 * max_ctas();
  float* part = nullptr;
  if (a->dbias) {
    const int rc = det_alloc((size_t)grid * a->C * sizeof(float), st, &part);
    if (rc) return rc;
  }
  softmax_ce_bwd_kernel<<<grid, 256, 0, st>>>(*a, part);
  if (a->dbias) {
    const int rc = det_reduce_launch(part, grid, a->C, a->dbias, st);
    if (rc) return rc;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "softmax_ce bwd: %s", cudaGetErrorString(e));
  return 0;
}

}  // namespace yamb
