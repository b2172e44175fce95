// Instance normalisation of the non-local block (nl_norm: nn.InstanceNorm, reference
// models/mobilenet_base.py:149-156, :472-481), training mode, on NHWC bf16 [N*HW][ld] matrices:
//   in_fwd  per-(n, c) statistics over the HW pixels of one sample -> y = gamma*xhat + beta
//           (+ residual + residual2), mean / invstd [N][C] for the backward, running statistics
//   in_bwd  per-(n, c) sums of dy and dy*xhat -> dh, dgamma / dbeta summed over the samples
// One CTA owns one (sample, 64-channel chunk): its statistics never leave the CTA, so a pass over
// the chunk's pixels computes them and a second pass applies them (the second read hits L2).
// Within a CTA each thread owns one 8-channel group and a strided set of pixels; its fp32 partial
// sums are combined in double in thread order.  What crosses samples (running statistics, dgamma,
// dbeta) is written per sample into a stream-ordered scratch and added in sample order by the last
// CTA (threadfence + counter, bn_finalize.cuh): no float atomics, the same bits on every run.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "bn_finalize.cuh"
#include "host_util.h"
#include "prims.cuh"

namespace yamb {
namespace {

constexpr int kThreads = 256;
constexpr int kChunk = 64;        // channels per CTA: 8 groups of 8
constexpr int kUnroll = 4;        // 16-byte loads in flight per thread

__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  v[0] = bf16lo(u.x); v[1] = bf16hi(u.x); v[2] = bf16lo(u.y); v[3] = bf16hi(u.y);
  v[4] = bf16lo(u.z); v[5] = bf16hi(u.z); v[6] = bf16lo(u.w); v[7] = bf16hi(u.w);
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&v)[8]) {
  *reinterpret_cast<uint4*>(p) = make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]),
                                            pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
}

// CTA blockIdx.x owns sample n = blockIdx.x / chunks and channel chunk blockIdx.x % chunks (a 1-D
// grid: arrive_last counts gridDim.x CTAs).  Thread layout over the chunk: CG (<= 8) channel
// groups x PX pixel lanes.
struct Lane {
  int n, chunk, CG, PX, cg, px, c0;
  bool active;
};
__device__ __forceinline__ Lane lane_of(int C) {
  Lane l;
  const int chunks = (C + kChunk - 1) / kChunk;
  l.n = blockIdx.x / chunks;
  l.chunk = blockIdx.x % chunks;
  const int groups = C / 8 - l.chunk * (kChunk / 8);
  l.CG = groups < kChunk / 8 ? groups : kChunk / 8;
  l.PX = kThreads / l.CG;
  l.cg = threadIdx.x % l.CG;
  l.px = threadIdx.x / l.CG;
  l.active = l.px < l.PX;
  l.c0 = l.chunk * kChunk + l.cg * 8;
  return l;
}

// Sum the per-thread (a, b) of the PX pixel lanes of every channel group in lane order, in double.
// Result in tot[2][kChunk] (channel relative to the chunk).  All threads must call it.
__device__ __forceinline__ void cta_merge(const Lane& l, const float (&a)[8], const float (&b)[8],
                                          double (*tot)[kChunk]) {
  __shared__ float red[kThreads][17];
  if (l.active) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      red[threadIdx.x][e] = a[e];
      red[threadIdx.x][8 + e] = b[e];
    }
  }
  __syncthreads();
  if (threadIdx.x < l.CG) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      double sa = 0.0, sb = 0.0;
      for (int j = 0; j < l.PX; ++j) {
        sa += (double)red[threadIdx.x + j * l.CG][e];
        sb += (double)red[threadIdx.x + j * l.CG][8 + e];
      }
      tot[0][threadIdx.x * 8 + e] = sa;
      tot[1][threadIdx.x * 8 + e] = sb;
    }
  }
  __syncthreads();
}

}  // namespace

struct InFwdDev {
  int N, HW, C, ldh, ldr, ldr2, ldy;
  const __nv_bfloat16* h;
  const float *gamma, *beta;
  float eps, momentum;
  float *running_mean, *running_var;
  float *mean, *invstd;
  const __nv_bfloat16 *residual, *residual2;
  __nv_bfloat16* y;
  float* var_unbiased;          // scratch [N][C] when the running statistics are updated
  uint32_t* counter;
};

__global__ void __launch_bounds__(kThreads) in_fwd_kernel(const __grid_constant__ InFwdDev p) {
  __shared__ double tot[2][kChunk];
  __shared__ float s_scale[kChunk], s_shift[kChunk];
  const Lane l = lane_of(p.C);
  const int n = l.n;
  const long long row0 = (long long)n * p.HW;
  // pass 1: sums of d = h - K and d^2, K = the sample's first pixel (keeps E[d^2] - E[d]^2 from
  // cancelling when |mean| >> std)
  float K[8], s[8], q[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) s[e] = q[e] = K[e] = 0.f;
  if (l.active) {
    load8(p.h + row0 * p.ldh + l.c0, K);
    int i = l.px;
    for (; i + (kUnroll - 1) * l.PX < p.HW; i += kUnroll * l.PX) {
      float v[kUnroll][8];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) load8(p.h + (row0 + i + u * l.PX) * p.ldh + l.c0, v[u]);
#pragma unroll
      for (int u = 0; u < kUnroll; ++u)
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float d = v[u][e] - K[e];
          s[e] += d;
          q[e] = fmaf(d, d, q[e]);
        }
    }
    for (; i < p.HW; i += l.PX) {
      float v[8];
      load8(p.h + (row0 + i) * p.ldh + l.c0, v);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float d = v[e] - K[e];
        s[e] += d;
        q[e] = fmaf(d, d, q[e]);
      }
    }
  }
  cta_merge(l, s, q, tot);
  if (threadIdx.x < l.CG) {
    const double inv_hw = 1.0 / (double)p.HW;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int cc = threadIdx.x * 8 + e, c = l.chunk * kChunk + cc;
      const double md = tot[0][cc] * inv_hw;
      double var = tot[1][cc] * inv_hw - md * md;
      if (var < 0.0) var = 0.0;
      const float mean = (float)((double)K[e] + md);
      const float invstd = (float)(1.0 / sqrt(var + (double)p.eps));
      const float g = p.gamma ? p.gamma[c] : 1.f;
      const float b = p.beta ? p.beta[c] : 0.f;
      const float sc = g * invstd;
      s_scale[cc] = sc;
      s_shift[cc] = b - mean * sc;
      p.mean[(size_t)n * p.C + c] = mean;
      p.invstd[(size_t)n * p.C + c] = invstd;
      if (p.var_unbiased)
        p.var_unbiased[(size_t)n * p.C + c] = (float)(var * ((double)p.HW / (double)(p.HW - 1)));
    }
  }
  __syncthreads();
  // pass 2: y = scale*h + shift (+ residual) (+ residual2), the order of yamb_bn_apply_fwd
  if (l.active) {
    const int cc = l.cg * 8;
    float sc[8], sh[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      sc[e] = s_scale[cc + e];
      sh[e] = s_shift[cc + e];
    }
    for (int i = l.px; i < p.HW; i += l.PX) {
      const long long r = row0 + i;
      float v[8];
      load8(p.h + r * p.ldh + l.c0, v);
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = fmaf(sc[e], v[e], sh[e]);
      if (p.residual) {
        float a[8];
        load8(p.residual + r * p.ldr + l.c0, a);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] += a[e];
      }
      if (p.residual2) {
        float a[8];
        load8(p.residual2 + r * p.ldr2 + l.c0, a);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] += a[e];
      }
      store8(p.y + r * p.ldy + l.c0, v);
    }
  }
  // running statistics: the last CTA averages the per-sample statistics in sample order
  if (p.var_unbiased == nullptr) return;
  if (arrive_last(p.counter)) {
    const float m = p.momentum;
    const double inv_n = 1.0 / (double)p.N;
    for (int c = threadIdx.x; c < p.C; c += kThreads) {
      double sm = 0.0, sv = 0.0;
      for (int k = 0; k < p.N; ++k) {
        sm += (double)__ldcg(p.mean + (size_t)k * p.C + c);
        sv += (double)__ldcg(p.var_unbiased + (size_t)k * p.C + c);
      }
      p.running_mean[c] = (1.f - m) * p.running_mean[c] + m * (float)(sm * inv_n);
      p.running_var[c] = (1.f - m) * p.running_var[c] + m * (float)(sv * inv_n);
    }
    __syncthreads();
    if (threadIdx.x == 0) *p.counter = 0;
  }
}

struct InBwdDev {
  int N, HW, C, ldh, lddy, lddh;
  const __nv_bfloat16 *dy, *h;
  const float* gamma;
  const float *mean, *invstd;
  float *dgamma, *dbeta;
  __nv_bfloat16* dh;
  float* slabs;                 // scratch [N][2][C]: sum(dy*xhat), sum(dy) per sample
  uint32_t* counter;
};

__global__ void __launch_bounds__(kThreads) in_bwd_kernel(const __grid_constant__ InBwdDev p) {
  __shared__ double tot[2][kChunk];
  __shared__ float s_a[kChunk], s_m1[kChunk], s_m2[kChunk];
  const Lane l = lane_of(p.C);
  const int n = l.n;
  const long long row0 = (long long)n * p.HW;
  float mu[8], rs[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) mu[e] = rs[e] = 0.f;
  if (l.active) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      mu[e] = p.mean[(size_t)n * p.C + l.c0 + e];
      rs[e] = p.invstd[(size_t)n * p.C + l.c0 + e];
    }
  }
  // pass 1: sum(dy), sum(dy * (h - mu))
  float s[8], q[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) s[e] = q[e] = 0.f;
  if (l.active) {
    int i = l.px;
    for (; i + (kUnroll - 1) * l.PX < p.HW; i += kUnroll * l.PX) {
      float g[kUnroll][8], v[kUnroll][8];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        load8(p.dy + (row0 + i + u * l.PX) * p.lddy + l.c0, g[u]);
        load8(p.h + (row0 + i + u * l.PX) * p.ldh + l.c0, v[u]);
      }
#pragma unroll
      for (int u = 0; u < kUnroll; ++u)
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          s[e] += g[u][e];
          q[e] = fmaf(g[u][e], v[u][e] - mu[e], q[e]);
        }
    }
    for (; i < p.HW; i += l.PX) {
      float g[8], v[8];
      load8(p.dy + (row0 + i) * p.lddy + l.c0, g);
      load8(p.h + (row0 + i) * p.ldh + l.c0, v);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        s[e] += g[e];
        q[e] = fmaf(g[e], v[e] - mu[e], q[e]);
      }
    }
  }
  cta_merge(l, s, q, tot);
  if (threadIdx.x < l.CG) {
    const double inv_hw = 1.0 / (double)p.HW;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int cc = threadIdx.x * 8 + e, c = l.chunk * kChunk + cc;
      const float r = p.invstd[(size_t)n * p.C + c];
      const double sdy = tot[0][cc], sdx = tot[1][cc] * (double)r;   // sum(dy), sum(dy*xhat)
      const float g = p.gamma ? p.gamma[c] : 1.f;
      s_a[cc] = g * r;
      s_m1[cc] = (float)(sdy * inv_hw);
      s_m2[cc] = (float)(sdx * inv_hw);
      if (p.slabs) {
        p.slabs[(size_t)n * 2 * p.C + c] = (float)sdx;
        p.slabs[(size_t)n * 2 * p.C + p.C + c] = (float)sdy;
      }
    }
  }
  __syncthreads();
  // pass 2: dh = a * (dy - m1 - xhat * m2)
  if (l.active) {
    const int cc = l.cg * 8;
    float a[8], m1[8], m2[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      a[e] = s_a[cc + e];
      m1[e] = s_m1[cc + e];
      m2[e] = s_m2[cc + e];
    }
    for (int i = l.px; i < p.HW; i += l.PX) {
      const long long r = row0 + i;
      float g[8], v[8];
      load8(p.dy + r * p.lddy + l.c0, g);
      load8(p.h + r * p.ldh + l.c0, v);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float xhat = (v[e] - mu[e]) * rs[e];
        v[e] = a[e] * (g[e] - m1[e] - xhat * m2[e]);
      }
      store8(p.dh + r * p.lddh + l.c0, v);
    }
  }
  // dgamma / dbeta: the last CTA adds the per-sample sums in sample order
  if (p.slabs == nullptr) return;
  if (arrive_last(p.counter)) {
    for (int c = threadIdx.x; c < p.C; c += kThreads) {
      double sg = 0.0, sb = 0.0;
      for (int k = 0; k < p.N; ++k) {
        sg += (double)__ldcg(p.slabs + (size_t)k * 2 * p.C + c);
        sb += (double)__ldcg(p.slabs + (size_t)k * 2 * p.C + p.C + c);
      }
      if (p.dgamma) p.dgamma[c] += (float)sg;
      if (p.dbeta) p.dbeta[c] += (float)sb;
    }
    __syncthreads();
    if (threadIdx.x == 0) *p.counter = 0;
  }
}

static bool ld_ok(int ld, int C) { return ld >= C && ld % 8 == 0; }

int in_fwd_launch(const yamb_in_fwd* a, cudaStream_t st) {
  if (!a || a->N <= 0 || a->N > 65535 || a->HW < 2 || a->C <= 0 || a->C % 8 || !ld_ok(a->ldh, a->C) ||
      !ld_ok(a->ldy, a->C) || !a->h || !a->y || !a->mean || !a->invstd ||
      (a->residual && !ld_ok(a->ldr, a->C)) || (a->residual2 && !ld_ok(a->ldr2, a->C)))
    return set_error(YAMB_EINVAL, "instance_norm_fwd: shape (N %d, HW %d, C %d; HW >= 2, C %% 8 == 0)",
                     a ? a->N : 0, a ? a->HW : 0, a ? a->C : 0);
  const bool update = a->running_mean && a->running_var && a->momentum != 0.f;
  if (update && !a->counter) return set_error(YAMB_EINVAL, "instance_norm_fwd: counter is NULL");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  InFwdDev p;
  p.N = a->N; p.HW = a->HW; p.C = a->C;
  p.ldh = a->ldh; p.ldr = a->ldr; p.ldr2 = a->ldr2; p.ldy = a->ldy;
  p.h = (const __nv_bfloat16*)a->h;
  p.gamma = a->gamma; p.beta = a->beta; p.eps = a->eps; p.momentum = a->momentum;
  p.running_mean = a->running_mean; p.running_var = a->running_var;
  p.mean = a->mean; p.invstd = a->invstd;
  p.residual = (const __nv_bfloat16*)a->residual;
  p.residual2 = (const __nv_bfloat16*)a->residual2;
  p.y = (__nv_bfloat16*)a->y;
  p.var_unbiased = nullptr;
  p.counter = a->counter;
  if (update) {
    int rc = det_alloc((size_t)a->N * a->C * sizeof(float), st, &p.var_unbiased);
    if (rc) return rc;
  }
  const int grid = (a->C + kChunk - 1) / kChunk * a->N;
  in_fwd_kernel<<<grid, kThreads, 0, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (update) {
    int rc = det_free(p.var_unbiased, st);
    if (e == cudaSuccess && rc) return rc;
  }
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "instance_norm_fwd: %s", cudaGetErrorString(e));
  return 0;
}

int in_bwd_launch(const yamb_in_bwd* a, cudaStream_t st) {
  if (!a || a->N <= 0 || a->N > 65535 || a->HW < 2 || a->C <= 0 || a->C % 8 || !ld_ok(a->ldh, a->C) ||
      !ld_ok(a->lddy, a->C) || !ld_ok(a->lddh, a->C) || !a->dy || !a->h || !a->dh || !a->mean ||
      !a->invstd)
    return set_error(YAMB_EINVAL, "instance_norm_bwd: shape (N %d, HW %d, C %d; HW >= 2, C %% 8 == 0)",
                     a ? a->N : 0, a ? a->HW : 0, a ? a->C : 0);
  const bool grads = a->dgamma || a->dbeta;
  if (grads && !a->counter) return set_error(YAMB_EINVAL, "instance_norm_bwd: counter is NULL");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  InBwdDev p;
  p.N = a->N; p.HW = a->HW; p.C = a->C;
  p.ldh = a->ldh; p.lddy = a->lddy; p.lddh = a->lddh;
  p.dy = (const __nv_bfloat16*)a->dy; p.h = (const __nv_bfloat16*)a->h;
  p.gamma = a->gamma; p.mean = a->mean; p.invstd = a->invstd;
  p.dgamma = a->dgamma; p.dbeta = a->dbeta;
  p.dh = (__nv_bfloat16*)a->dh;
  p.slabs = nullptr;
  p.counter = a->counter;
  if (grads) {
    int rc = det_alloc((size_t)a->N * 2 * a->C * sizeof(float), st, &p.slabs);
    if (rc) return rc;
  }
  const int grid = (a->C + kChunk - 1) / kChunk * a->N;
  in_bwd_kernel<<<grid, kThreads, 0, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (grads) {
    int rc = det_free(p.slabs, st);
    if (e == cudaSuccess && rc) return rc;
  }
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "instance_norm_bwd: %s", cudaGetErrorString(e));
  return 0;
}

}  // namespace yamb
