// Per-channel statistics plumbing shared by every producer kernel (pointwise GEMM, depthwise).
//
// A producer CTA accumulates per-channel partial sums in registers (fp32, fixed order) and hands
// them on through shared memory and the global accumulator partials[stat][C] with fire-and-forget
// reductions (red.add — a serial reduction of a [CTAs][2][C] table by the last CTA cost 15-30 us
// per BatchNorm, measured).  Everything that crosses warps or CTAs is accumulated in DOUBLE
// (stat_t): the order of those additions is not fixed, and in fp32 their reordering changed the
// BatchNorm coefficients in the last bits, which bf16 rounding flips downstream amplified to a
// 1e-3 run-to-run difference of the loss; fp64 sums of fp32 partials are reproducible to 1e-16
// relative, i.e. the fp32 mean / invstd they are rounded to are the same bits run after run
// (barring an exact rounding tie).  It also takes the E[x^2]-mean^2 cancellation out of fp32.
// The LAST CTA to finish (threadfence + counter) reads the 2C totals, returns the accumulator
// to zero (it must be zero on entry) and runs the BatchNorm bookkeeping of nn.BatchNorm2d
// (reference: models/mobilenet_base.py:203,417 -> torch.nn.BatchNorm2d semantics):
//   forward : mean / biased var -> scale, shift (what the consumer kernel applies), saved
//             mean/invstd, running stats with UNBIASED var, momentum or cumulative (momentum<0).
//   backward: sum(dz), sum(dz*xhat) -> dgamma, dbeta and the affine coefficients
//             dh = ca*dz + cb*h + cc that the consumer kernel applies on load.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/yamb200.h"

namespace yamb {

typedef double stat_t;   // cross-warp / cross-CTA statistics accumulator

// Count this CTA as finished; true in the LAST CTA of the grid (whose later reads see every other
// CTA's earlier global reductions).  Must be called by ALL threads of the CTA.
__device__ __forceinline__ bool arrive_last(uint32_t* counter) {
  __shared__ uint32_t s_is_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t prev = atomicAdd(counter, 1u);
    s_is_last = (prev == gridDim.x - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (s_is_last) __threadfence();
  return s_is_last != 0;
}

// arrive_last for a CTA that is one of `nblk` CTAs counted on `counter` (a range of a grouped grid)
__device__ __forceinline__ bool arrive_last_of(uint32_t* counter, unsigned nblk) {
  __shared__ uint32_t s_is_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t prev = atomicAdd(counter, 1u);
    s_is_last = (prev == nblk - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (s_is_last) __threadfence();
  return s_is_last != 0;
}

// Add this CTA's partials (s_part: [2][C] in shared memory) to the global accumulator and return
// true in the last CTA.  Must be called by ALL threads of the CTA.
__device__ __forceinline__ bool publish_partials(const stat_t* s_part, int C, stat_t* partials,
                                                 uint32_t* counter) {
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
    stat_t v = s_part[i];
    if (v != 0.0) atomicAdd(partials + i, v);  // result unused -> RED.E.ADD.F64
  }
  return arrive_last(counter);
}

// Merge the per-thread partial sums (s, q: 8 channels each) of the threads of a CTA that own the
// same 8-channel group (tid = px * CG + cg, px < PX) into the CTA's statistics slots WITHOUT
// atomics: staged through shared memory and summed in pixel-lane order by the px == 0 thread, in
// double.  (Shared-memory double atomics are CAS loops; PX threads contending for every slot cost
// bn_reduce 20 %.)  Must be called by ALL threads of the CTA; `active` = this thread holds sums.
__device__ __forceinline__ void cta_stats_merge(stat_t* s_part, int C, int CG, int PX, int cg, int px,
                                                bool active, const float (&s)[8],
                                                const float (&q)[8]) {
  __shared__ float red[256][17];
  if (active) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      red[threadIdx.x][e] = s[e];
      red[threadIdx.x][8 + e] = q[e];
    }
  }
  __syncthreads();
  if (active && px == 0) {
    const int c0 = cg * 8;
    const int base = threadIdx.x;              // = cg (relative to this pass) when px == 0
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      stat_t a = 0.0, b = 0.0;
      for (int j = 0; j < PX; ++j) {
        a += (stat_t)red[base + j * CG][e];
        b += (stat_t)red[base + j * CG][8 + e];
      }
      s_part[c0 + e] += a;
      s_part[C + c0 + e] += b;
    }
  }
  __syncthreads();
}

// Read-and-clear one total (L2 is the point of coherence for the reductions above).
__device__ __forceinline__ double take_total(stat_t* p) {
  double v = __ldcg(p);
  __stcg(p, 0.0);
  return v;
}

__device__ __forceinline__ void bn_fwd_finalize(const yamb_bn_fwd& f, int C) {
  const double inv_count = 1.0 / (double)f.count;
  float factor = f.momentum;
  if (f.num_batches_tracked != nullptr) {
    long long nbt = *f.num_batches_tracked + 1;
    if (f.momentum < 0.f) factor = 1.0f / (float)nbt;  // momentum=None: cumulative average
    __syncthreads();
    if (threadIdx.x == 0) *f.num_batches_tracked = nbt;
  }
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double s = take_total(f.partials + c), q = take_total(f.partials + C + c);
    double mean = s * inv_count;
    double var = q * inv_count - mean * mean;
    if (var < 0.0) var = 0.0;
    float invstd = (float)(1.0 / sqrt(var + (double)f.eps));
    float g = f.gamma ? f.gamma[c] : 1.f;
    float b = f.beta ? f.beta[c] : 0.f;
    float sc = g * invstd;
    f.scale[c] = sc;
    f.shift[c] = b - (float)mean * sc;
    if (f.mean) f.mean[c] = (float)mean;
    if (f.invstd) f.invstd[c] = invstd;
    if (f.running_mean) {
      double unbiased = f.count > 1 ? var * ((double)f.count / (double)(f.count - 1)) : var;
      f.running_mean[c] = (1.f - factor) * f.running_mean[c] + factor * (float)mean;
      f.running_var[c] = (1.f - factor) * f.running_var[c] + factor * (float)unbiased;
    }
  }
}

// channel c of the backward finalize from its totals s = sum(dz), q = sum(dz * xhat);
// inv_count = 1 / f.count
__device__ __forceinline__ void bn_bwd_coeffs(const yamb_bn_bwd& f, int c, double s, double q,
                                              double inv_count) {
  if (f.dgamma) f.dgamma[c] += (float)q;
  if (f.dbeta) f.dbeta[c] += (float)s;
  float g = f.gamma ? f.gamma[c] : 1.f;
  float r = f.invstd[c];
  float mu = f.mean[c];
  float sc = g * r;
  float m1 = (float)(s * inv_count), m2 = (float)(q * inv_count);
  f.ca[c] = sc;
  f.cb[c] = f.use_batch_stats ? -sc * r * m2 : 0.f;
  f.cc[c] = f.use_batch_stats ? sc * (mu * r * m2 - m1) : 0.f;
}

__device__ __forceinline__ void bn_bwd_finalize(const yamb_bn_bwd& f, int C) {
  const double inv_count = 1.0 / (double)f.count;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double s = take_total(f.partials + c), q = take_total(f.partials + C + c);
    bn_bwd_coeffs(f, c, s, q, inv_count);
  }
}

}  // namespace yamb
