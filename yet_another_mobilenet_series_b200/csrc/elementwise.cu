// HBM-bound per-channel kernels on [pixels, channels] bf16 matrices, sm_90a:
//   bn_apply   y = act(scale[c]*h + shift[c]) (+ residual)        — pw_bn + skip connection of
//              the block (reference models/mobilenet_base.py:448-450, :340-341) and the
//              ConvBNReLU tails (:203)
//   bn_reduce  sum(dy), sum(dy*xhat) per channel + BatchNorm-backward finalize (last CTA)
//   se_pool / se_gate / se_bwd: Squeeze-and-Excitation pieces (reference :110-113)
// 16-byte vector accesses, consecutive threads -> consecutive channel groups, then pixels.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "bn_finalize.cuh"
#include "host_util.h"
#include "prims.cuh"

namespace yamb {

struct BnApplyDev {
  long long M;
  int C, ldh, ldr, ldy;
  const __nv_bfloat16* h;
  const float *scale, *shift;
  int act;
  const __nv_bfloat16* residual;
  __nv_bfloat16* y;
  // optional per-(sample, channel) gate (SE): y *= gate[n][c], n = row / rows_per_sample
  const float* gate;
  long long rows_per_sample;
  const __nv_bfloat16* residual2;
  int ldr2;
};

__global__ void __launch_bounds__(256) bn_apply_kernel(const __grid_constant__ BnApplyDev p) {
  const int CG = p.C / 8;
  const long long total = p.M * CG;
  const ActParam ap = make_act(p.act);
  // (row, channel group) advance incrementally: one 64-bit division per thread instead of one per
  // 16-byte vector (a ~70-instruction sequence next to ~40 instructions of useful work)
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long d_row = stride / CG;
  const int d_cg = (int)(stride % CG);
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long row = i / CG;
  int cgi = (int)(i % CG);
  for (; i < total; i += stride, row += d_row, cgi += d_cg) {
    if (cgi >= CG) { cgi -= CG; ++row; }
    const int c0 = cgi * 8;
    float v[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(p.h + row * p.ldh + c0)), v);
    const float4 s0 = __ldg(reinterpret_cast<const float4*>(p.scale + c0));
    const float4 s1 = __ldg(reinterpret_cast<const float4*>(p.scale + c0 + 4));
    const float4 t0 = __ldg(reinterpret_cast<const float4*>(p.shift + c0));
    const float4 t1 = __ldg(reinterpret_cast<const float4*>(p.shift + c0 + 4));
    const float sc[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    const float sh[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = fmaf(sc[e], v[e], sh[e]);
    act_vec<8>(v, ap);
    if (p.gate) {
      const float* g = p.gate + (row / p.rows_per_sample) * p.C + c0;
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] *= __ldg(g + e);
    }
    if (p.residual) {
      float r[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(p.residual + row * p.ldr + c0)), r);
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] += r[e];
    }
    if (p.residual2) {
      float r[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(p.residual2 + row * p.ldr2 + c0)), r);
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] += r[e];
    }
    *reinterpret_cast<uint4*>(p.y + row * p.ldy + c0) = pack8(v);
  }
}

struct BnReduceDev {
  long long M;
  int C, lddy, ldh;
  const __nv_bfloat16* dy;
  const __nv_bfloat16* h;
  yamb_bn_bwd bn;
  const float *z_scale, *z_shift;   // optional activation after the BatchNorm: dz = dy*act'(z)
  int z_act;
};

// sum(dy), sum(dy * xhat) with xhat = (h - mean) * invstd; thread owns one 8-channel group.
__global__ void __launch_bounds__(256) bn_reduce_kernel(const __grid_constant__ BnReduceDev p) {
  extern __shared__ stat_t s_part[];  // [2][C], double
  const int CG = p.C / 8;
  const int PX = 256 / CG > 0 ? 256 / CG : 1;
  for (int i = threadIdx.x; i < 2 * p.C; i += blockDim.x) s_part[i] = 0.0;
  __syncthreads();
  // channel groups beyond 256 are covered by looping cg
  for (int cgb = 0; cgb < CG; cgb += 256) {
    const int cg = cgb + (CG >= 256 ? threadIdx.x : threadIdx.x % CG);
    const int px = CG >= 256 ? 0 : threadIdx.x / CG;
    const bool active = cg < CG && px < PX;
    float s[8], q[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) s[e] = q[e] = 0.f;
    if (active) {
      const int c0 = cg * 8;
      float mu[8], rs[8], zs[8], zt[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        mu[e] = __ldg(p.bn.mean + c0 + e);
        rs[e] = __ldg(p.bn.invstd + c0 + e);
        zs[e] = p.z_scale ? __ldg(p.z_scale + c0 + e) : 1.f;
        zt[e] = p.z_scale ? __ldg(p.z_shift + c0 + e) : 0.f;
        s[e] = q[e] = 0.f;
      }
      const ActParam zap = make_act(p.z_scale ? p.z_act : ACT_NONE);
      // 4 rows (8 independent 16-byte loads) in flight per thread: with one row per iteration the
      // kernel ran at 1.5 TB/s, latency-bound
      const long long rstep = (long long)gridDim.x * PX;
      for (long long row = (long long)blockIdx.x * PX + px; row < p.M; row += 4 * rstep) {
        uint4 ud[4], uh[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const long long r2 = row + j * rstep;
          ud[j] = make_uint4(0u, 0u, 0u, 0u);
          uh[j] = make_uint4(0u, 0u, 0u, 0u);
          if (r2 < p.M) {
            ud[j] = __ldg(reinterpret_cast<const uint4*>(p.dy + r2 * p.lddy + c0));
            uh[j] = __ldg(reinterpret_cast<const uint4*>(p.h + r2 * p.ldh + c0));
          }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float d[8], hv[8];
          unpack8(ud[j], d);     // a row past M contributes dy = 0
          unpack8(uh[j], hv);
          if (p.z_scale) {
            float z[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) z[e] = fmaf(zs[e], hv[e], zt[e]);
            act_bwd_vec<8>(d, z, zap, p.z_act);
          }
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            s[e] += d[e];
            q[e] = fmaf(d[e], (hv[e] - mu[e]) * rs[e], q[e]);
          }
        }
      }
    }
    cta_stats_merge(s_part, p.C, CG >= 256 ? 256 : CG, PX, cg, px, active, s, q);
  }
  __syncthreads();
  if (publish_partials(s_part, p.C, p.bn.partials, p.bn.counter)) {
    bn_bwd_finalize(p.bn, p.C);
    __syncthreads();
    if (threadIdx.x == 0) *p.bn.counter = 0;
  }
}

// Stand-alone BatchNorm of a convolution run elsewhere (stem / head ConvBNReLU): per-channel
// sum(h), sum(h^2) + BatchNorm forward finalize (last CTA).  Same thread layout as bn_reduce.
struct BnStatsDev {
  long long M;
  int C, ldh;
  const __nv_bfloat16* h;
  yamb_bn_fwd bn;
};
__global__ void __launch_bounds__(256) bn_stats_kernel(const __grid_constant__ BnStatsDev p) {
  extern __shared__ stat_t s_part[];  // [2][C], double
  const int CG = p.C / 8;
  const int PX = 256 / CG > 0 ? 256 / CG : 1;
  for (int i = threadIdx.x; i < 2 * p.C; i += blockDim.x) s_part[i] = 0.0;
  __syncthreads();
  for (int cgb = 0; cgb < CG; cgb += 256) {
    const int cg = cgb + (CG >= 256 ? threadIdx.x : threadIdx.x % CG);
    const int px = CG >= 256 ? 0 : threadIdx.x / CG;
    const bool active = cg < CG && px < PX;
    float s[8], q[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) s[e] = q[e] = 0.f;
    if (active) {
      const int c0 = cg * 8;
      const long long rstep = (long long)gridDim.x * PX;
      for (long long row = (long long)blockIdx.x * PX + px; row < p.M; row += 4 * rstep) {
        uint4 uh[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const long long r2 = row + j * rstep;
          uh[j] = r2 < p.M ? __ldg(reinterpret_cast<const uint4*>(p.h + r2 * p.ldh + c0))
                           : make_uint4(0u, 0u, 0u, 0u);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float hv[8];
          unpack8(uh[j], hv);
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            s[e] += hv[e];
            q[e] = fmaf(hv[e], hv[e], q[e]);
          }
        }
      }
    }
    cta_stats_merge(s_part, p.C, CG >= 256 ? 256 : CG, PX, cg, px, active, s, q);
  }
  __syncthreads();
  if (publish_partials(s_part, p.C, p.bn.partials, p.bn.counter)) {
    bn_fwd_finalize(p.bn, p.C);
    __syncthreads();
    if (threadIdx.x == 0) *p.bn.counter = 0;
  }
}

// dh = ca*dz + cb*h + cc,  dz = dy * act'(z_scale*h + z_shift)
struct BnBwdApplyDev {
  long long M;
  int C, lddy, ldh, lddh;
  const __nv_bfloat16* dy;
  const __nv_bfloat16* h;
  const float *z_scale, *z_shift;
  int z_act;
  const float *ca, *cb, *cc;
  __nv_bfloat16* dh;
};
// Thread layout of bn_reduce: a thread owns one 8-channel group (its coefficients stay in registers)
// and walks pixel rows with 4 rows (8 independent 16-byte loads) in flight; one load pair per
// iteration left the kernel latency-bound.  The arithmetic is that of the GEMM loaders' two-source
// transform (gxform_panel<2>: fmaf(ca, dy, fmaf(cb, h, cc)), RN to bf16), so a GEMM that reads
// this dh gets the operand bits the transform would have formed.
__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(const __grid_constant__ BnBwdApplyDev p) {
  const int CG = p.C / 8;
  const int PX = 256 / CG > 0 ? 256 / CG : 1;
  const ActParam zap = make_act(p.z_scale ? p.z_act : ACT_NONE);
  // channel groups beyond 256 are covered by looping cg
  for (int cgb = 0; cgb < CG; cgb += 256) {
    const int cg = cgb + (CG >= 256 ? threadIdx.x : threadIdx.x % CG);
    const int px = CG >= 256 ? 0 : threadIdx.x / CG;
    if (cg >= CG || px >= PX) continue;
    const int c0 = cg * 8;
    float ca[8], cb[8], cc[8], zs[8], zt[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      ca[e] = __ldg(p.ca + c0 + e);
      cb[e] = __ldg(p.cb + c0 + e);
      cc[e] = __ldg(p.cc + c0 + e);
      zs[e] = p.z_scale ? __ldg(p.z_scale + c0 + e) : 1.f;
      zt[e] = p.z_scale ? __ldg(p.z_shift + c0 + e) : 0.f;
    }
    const long long rstep = (long long)gridDim.x * PX;
    for (long long row = (long long)blockIdx.x * PX + px; row < p.M; row += 4 * rstep) {
      uint4 ud[4], uh[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const long long r2 = row + j * rstep;
        ud[j] = make_uint4(0u, 0u, 0u, 0u);
        uh[j] = make_uint4(0u, 0u, 0u, 0u);
        if (r2 < p.M) {
          ud[j] = __ldg(reinterpret_cast<const uint4*>(p.dy + r2 * p.lddy + c0));
          uh[j] = __ldg(reinterpret_cast<const uint4*>(p.h + r2 * p.ldh + c0));
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const long long r2 = row + j * rstep;
        float d[8], hv[8];
        unpack8(ud[j], d);
        unpack8(uh[j], hv);
        if (p.z_scale) {
          float z[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) z[e] = fmaf(zs[e], hv[e], zt[e]);
          act_bwd_vec<8>(d, z, zap, p.z_act);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) d[e] = fmaf(ca[e], d[e], fmaf(cb[e], hv[e], cc[e]));
        if (r2 < p.M) *reinterpret_cast<uint4*>(p.dh + r2 * p.lddh + c0) = pack8(d);
      }
    }
  }
}

// ---- Squeeze-and-Excitation ----------------------------------------------------------------------
// pooled[n][c] = mean over HW of act(scale*h+shift)  (a2 is never materialised).
struct SePoolDev {
  int N, HW, C, ldh;
  const __nv_bfloat16* h;
  const float *scale, *shift;
  int act;
  float* pooled;  // [pixel chunks][N][out_ld] slabs (slab = pixel-chunk stride)
  int out_ld;
  long long slab;
};
// grid (pixel chunks, N); thread = (8-channel group cg, pixel lane px): whole 16-byte-per-lane rows
// are read (every lane busy whatever C is), 4 rows in flight per thread, lanes reduced through
// shared memory, then one plain store per (n, c) into the slab of this CTA's pixel chunk
// (out + blockIdx.x * slab); the launcher adds the slabs in slab order.
// With kStats (se_bwd_stats) the same walk also takes the BatchNorm-2 backward sums of SeStatsDev
// into double slabs [pixel chunk][4][st->plane], added over the pixel lanes in lane order.
struct SeStatsDev {
  const float *mean, *invstd;   // [C] BatchNorm-2 statistics
  double* sums;                 // slab of pixel chunk b: sums + b * 4 * plane; [4][N][out_ld]
  long long plane;              // N * out_ld
};
template <bool kBwd, bool kStats = false>
__device__ __forceinline__ void se_rows_reduce(int N, int HW, int C, const __nv_bfloat16* h, int ldh,
                                               const __nv_bfloat16* dy, int ldd, const float* scale,
                                               const float* shift, int act, float out_scale,
                                               float* out, int out_ld, long long slab,
                                               const SeStatsDev* st = nullptr) {
  __shared__ float red[256][kStats ? 41 : 9];
  const int CG = C / 8;
  const int PX = 256 / CG;                       // pixel lanes (host guarantees CG <= 256)
  const int cg = threadIdx.x % CG, px = threadIdx.x / CG;
  const int n = blockIdx.y;
  const int rows_per = (HW + gridDim.x - 1) / gridDim.x;
  const int r0 = blockIdx.x * rows_per, r1 = min(HW, r0 + rows_per);
  float s[8];
  float sA[8], sB[8], sA2[8], sB2[8];   // kStats: A, B, A', B' (see yamb_se_bwd_stats)
#pragma unroll
  for (int e = 0; e < 8; ++e) s[e] = 0.f;
  if constexpr (kStats) {
#pragma unroll
    for (int e = 0; e < 8; ++e) sA[e] = sB[e] = sA2[e] = sB2[e] = 0.f;
  }
  if (px < PX) {
    const int c0 = cg * 8;
    const ActParam ap = make_act(act);
    float sc[8], sh[8], mu[8], rs[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { sc[e] = __ldg(scale + c0 + e); sh[e] = __ldg(shift + c0 + e); }
    if constexpr (kStats) {
#pragma unroll
      for (int e = 0; e < 8; ++e) { mu[e] = __ldg(st->mean + c0 + e); rs[e] = __ldg(st->invstd + c0 + e); }
    }
    const __nv_bfloat16* hb = h + (size_t)n * HW * ldh + c0;
    const __nv_bfloat16* db = kBwd ? dy + (size_t)n * HW * ldd + c0 : nullptr;
    auto body = [&](const uint4& hr, const uint4& dr) {
      float v[8];
      unpack8(hr, v);
      float hv[8], z[8];
      if constexpr (kStats) {
#pragma unroll
        for (int e = 0; e < 8; ++e) hv[e] = v[e];
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = fmaf(sc[e], v[e], sh[e]);
      if constexpr (kStats) {
#pragma unroll
        for (int e = 0; e < 8; ++e) z[e] = v[e];
      }
      act_vec<8>(v, ap);
      if (kBwd) {
        float d[8];
        unpack8(dr, d);
#pragma unroll
        for (int e = 0; e < 8; ++e) s[e] = fmaf(d[e], round_bf16(v[e]), s[e]);
        if constexpr (kStats) {
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            // act' and xhat as se_bwd_apply_kernel forms them
            const float g = act_bwd_rt(z[e], ap, act);
            const float xh = (hv[e] - mu[e]) * rs[e];
            const float t = d[e] * g;
            sA[e] += t;
            sB[e] += g;
            sA2[e] = fmaf(t, xh, sA2[e]);
            sB2[e] = fmaf(g, xh, sB2[e]);
          }
        }
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) s[e] += round_bf16(v[e]);
      }
    };
    int i = r0 + px;
    for (; i + 3 * PX < r1; i += 4 * PX) {
      uint4 hr[4], dr[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        hr[u] = __ldg(reinterpret_cast<const uint4*>(hb + (size_t)(i + u * PX) * ldh));
        dr[u] = kBwd ? __ldg(reinterpret_cast<const uint4*>(db + (size_t)(i + u * PX) * ldd))
                     : make_uint4(0u, 0u, 0u, 0u);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) body(hr[u], dr[u]);
    }
    for (; i < r1; i += PX)
      body(__ldg(reinterpret_cast<const uint4*>(hb + (size_t)i * ldh)),
           kBwd ? __ldg(reinterpret_cast<const uint4*>(db + (size_t)i * ldd)) : make_uint4(0u, 0u, 0u, 0u));
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) red[threadIdx.x][e] = s[e];
  if constexpr (kStats) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      red[threadIdx.x][8 + e] = sA[e];
      red[threadIdx.x][16 + e] = sB[e];
      red[threadIdx.x][24 + e] = sA2[e];
      red[threadIdx.x][32 + e] = sB2[e];
    }
  }
  __syncthreads();
  if (px == 0) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float t = 0.f;
      for (int j = 0; j < PX; ++j) t += red[j * CG + cg][e];
      out[(size_t)blockIdx.x * slab + (size_t)n * out_ld + cg * 8 + e] = t * out_scale;
    }
    if constexpr (kStats) {
      double* o = st->sums + (size_t)blockIdx.x * 4 * st->plane + (size_t)n * out_ld + cg * 8;
      for (int k = 0; k < 4; ++k) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          double t = 0.0;
          for (int j = 0; j < PX; ++j) t += (double)red[j * CG + cg][8 + 8 * k + e];
          o[(size_t)k * st->plane + e] = t;
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256) se_pool_kernel(const __grid_constant__ SePoolDev p) {
  se_rows_reduce<false>(p.N, p.HW, p.C, p.h, p.ldh, nullptr, 0, p.scale, p.shift, p.act,
                        1.f / (float)p.HW, p.pooled, p.out_ld, p.slab);
}

// dgate[n][c] = sum over HW of dY[n,hw,c] * round_bf16(act(scale*h + shift))  (SE backward, the
// gradient of x*gate w.r.t. gate; reference models/mobilenet_base.py:113 via autograd)
struct SeBwdReduceDev {
  int N, HW, C, ldd, ldh;
  const __nv_bfloat16* dy;
  const __nv_bfloat16* h;
  const float *scale, *shift;
  int act;
  float* dgate;  // [pixel chunks][N][out_ld] slabs, as SePoolDev::pooled
  int out_ld;
  long long slab;
};
__global__ void __launch_bounds__(256) se_bwd_reduce_kernel(const __grid_constant__ SeBwdReduceDev p) {
  se_rows_reduce<true>(p.N, p.HW, p.C, p.h, p.ldh, p.dy, p.ldd, p.scale, p.shift, p.act, 1.f,
                       p.dgate, p.out_ld, p.slab);
}

// dgate of se_bwd_reduce_kernel (the same bits) plus the BatchNorm-2 backward sums A, B, A', B'
// (yamb_se_bwd_stats), so that se_bn_bwd_finalize and dw_bwd_se_kernel replace se_bwd_apply.
struct SeBwdStatsDev {
  SeBwdReduceDev r;
  SeStatsDev st;
};
__global__ void __launch_bounds__(256) se_bwd_stats_kernel(const __grid_constant__ SeBwdStatsDev p) {
  se_rows_reduce<true, true>(p.r.N, p.r.HW, p.r.C, p.r.h, p.r.ldh, p.r.dy, p.r.ldd, p.r.scale,
                             p.r.shift, p.r.act, 1.f, p.r.dgate, p.r.out_ld, p.r.slab, &p.st);
}

// out[i] = sum over s = 0 .. nslab-1 of part[s * n + i], in that order (double slabs of
// se_bwd_stats_kernel)
__global__ void __launch_bounds__(256) se_sums_reduce_kernel(const double* __restrict__ part,
                                                             int nslab, long long n,
                                                             double* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    double s = 0.0;
    for (int k = 0; k < nslab; ++k) s += part[(size_t)k * n + i];
    out[i] = s;
  }
}

// BatchNorm-2 backward of one slice from the sums of se_bwd_stats_kernel and the SE FC backward's
// dpool: per channel sum(dz) = sum_n gate*A + dpool*B, sum(dz*xhat) = sum_n gate*A' + dpool*B'.
// A CTA owns 32 channels; its 8 sample lanes (warps) take n = lane, lane + 8, ... and are added in
// lane order, in double, before the finalize of bn_finalize.cuh.
struct SeBnFinalizeDev {
  int N, C, lds, ldg;
  const double* sums;
  const float *gate, *dpool;
  yamb_bn_bwd bn;
};
__global__ void __launch_bounds__(256) se_bn_bwd_finalize_kernel(const __grid_constant__ SeBnFinalizeDev p) {
  __shared__ double red[8][2][32];
  const int lane = threadIdx.x % 32, nl = threadIdx.x / 32;
  const int c = blockIdx.x * 32 + lane;
  double s = 0.0, q = 0.0;
  if (c < p.C) {
    const long long plane = (long long)p.N * p.lds;
    for (int n = nl; n < p.N; n += 8) {
      const double* a = p.sums + (size_t)n * p.lds + c;
      const double g = __ldg(p.gate + (size_t)n * p.ldg + c), d = __ldg(p.dpool + (size_t)n * p.ldg + c);
      s += g * __ldg(a) + d * __ldg(a + plane);
      q += g * __ldg(a + 2 * plane) + d * __ldg(a + 3 * plane);
    }
  }
  red[nl][0][lane] = s;
  red[nl][1][lane] = q;
  __syncthreads();
  if (nl == 0 && c < p.C) {
    for (int j = 1; j < 8; ++j) {
      s += red[j][0][lane];
      q += red[j][1][lane];
    }
    bn_bwd_coeffs(p.bn, c, s, q, 1.0 / (double)p.bn.count);
  }
}

// dz = (dY * gate[n][c] + dpool[n][c]) * act'(scale*h + shift)   (in place allowed: dz == dY)
// + BatchNorm-backward statistics sum(dz), sum(dz*xhat) and finalize (last CTA).
struct SeBwdApplyDev {
  long long M;
  int C, ldd, ldh, ldz;
  long long rows_per_sample;
  const __nv_bfloat16* dy;
  const __nv_bfloat16* h;
  const float *scale, *shift;
  int act;
  const float* gate;   // [N][C]
  const float* dpool;  // [N][C]  (already divided by HW)
  int ldg;             // row pitch of gate / dpool
  __nv_bfloat16* dz;
  yamb_bn_bwd bn;
};
__global__ void __launch_bounds__(256) se_bwd_apply_kernel(const __grid_constant__ SeBwdApplyDev p) {
  extern __shared__ stat_t s_part[];  // [2][C], double
  const int CG = p.C / 8;
  const int PX = 256 / CG > 0 ? 256 / CG : 1;
  for (int i = threadIdx.x; i < 2 * p.C; i += blockDim.x) s_part[i] = 0.0;
  __syncthreads();
  const ActParam ap = make_act(p.act);
  for (int cgb = 0; cgb < CG; cgb += 256) {
    const int cg = cgb + (CG >= 256 ? threadIdx.x : threadIdx.x % CG);
    const int px = CG >= 256 ? 0 : threadIdx.x / CG;
    const bool active = cg < CG && px < PX;
    float s[8], q[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) s[e] = q[e] = 0.f;
    if (active) {
      const int c0 = cg * 8;
      float sc[8], sh[8], mu[8], rs[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        sc[e] = __ldg(p.scale + c0 + e); sh[e] = __ldg(p.shift + c0 + e);
        mu[e] = __ldg(p.bn.mean + c0 + e); rs[e] = __ldg(p.bn.invstd + c0 + e);
        s[e] = q[e] = 0.f;
      }
      for (long long row = (long long)blockIdx.x * PX + px; row < p.M;
           row += (long long)gridDim.x * PX) {
        const long long n = (p.M < 0x7fffffffLL)
            ? (long long)((unsigned)row / (unsigned)p.rows_per_sample) : row / p.rows_per_sample;
        float d[8], hv[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(p.dy + row * p.ldd + c0)), d);
        unpack8(__ldg(reinterpret_cast<const uint4*>(p.h + row * p.ldh + c0)), hv);
        const float4* g4 = reinterpret_cast<const float4*>(p.gate + n * p.ldg + c0);
        const float4* d4 = reinterpret_cast<const float4*>(p.dpool + n * p.ldg + c0);
        const float4 ga = __ldg(g4), gb = __ldg(g4 + 1), pa = __ldg(d4), pb = __ldg(d4 + 1);
        const float gg[8] = {ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w};
        const float pp[8] = {pa.x, pa.y, pa.z, pa.w, pb.x, pb.y, pb.z, pb.w};
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float z = fmaf(sc[e], hv[e], sh[e]);
          d[e] = fmaf(d[e], gg[e], pp[e]) * act_bwd_rt(z, ap, p.act);
        }
        const uint4 o = pack8(d);
        *reinterpret_cast<uint4*>(p.dz + row * p.ldz + c0) = o;
        float r[8];
        unpack8(o, r);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          s[e] += r[e];
          q[e] = fmaf(r[e], (hv[e] - mu[e]) * rs[e], q[e]);
        }
      }
    }
    cta_stats_merge(s_part, p.C, CG >= 256 ? 256 : CG, PX, cg, px, active, s, q);
  }
  __syncthreads();
  if (publish_partials(s_part, p.C, p.bn.partials, p.bn.counter)) {
    bn_bwd_finalize(p.bn, p.C);
    __syncthreads();
    if (threadIdx.x == 0) *p.bn.counter = 0;
  }
}

// ---- launchers -----------------------------------------------------------------------------------
// A bf16 [rows][ld] operand that the kernels read or write 16 bytes (8 channels) at a time: present,
// ld >= C, rows of whole 16-byte vectors and a 16-byte aligned base.
static int check_bf16(const char* fn, const char* name, const void* p, int ld, int C) {
  if (!p) return set_error(YAMB_EINVAL, "%s: %s is NULL", fn, name);
  if (ld < C || ld % 8)
    return set_error(YAMB_EINVAL, "%s: row pitch of %s is %d, needs >= C = %d and a multiple of 8", fn,
                     name, ld, C);
  if (reinterpret_cast<uintptr_t>(p) & 15)
    return set_error(YAMB_EINVAL, "%s: %s must be 16-byte aligned", fn, name);
  return 0;
}

// bn_stats, bn_reduce and se_bwd_apply take 2*C doubles of dynamic shared memory (the CTA's
// statistics slots) on top of cta_stats_merge's static staging: from C = 1984 on they opt in.
static size_t stats_smem(int C) { return 2 * (size_t)C * sizeof(stat_t); }

int bn_apply_launch(const yamb_bn_apply* a, cudaStream_t st) {
  if (!a || a->M <= 0 || a->C <= 0 || (a->C % 8)) return set_error(YAMB_EINVAL, "bn_apply shape");
  int rc;
  if ((rc = check_bf16("bn_apply", "h", a->h, a->ldh, a->C)) ||
      (rc = check_bf16("bn_apply", "y", a->y, a->ldy, a->C)) ||
      (a->residual && (rc = check_bf16("bn_apply", "residual", a->residual, a->ldr, a->C))) ||
      (a->residual2 && (rc = check_bf16("bn_apply", "residual2", a->residual2, a->ldr2, a->C))))
    return rc;
  if (!a->scale || !a->shift ||
      ((reinterpret_cast<uintptr_t>(a->scale) | reinterpret_cast<uintptr_t>(a->shift)) & 15))
    return set_error(YAMB_EINVAL, "bn_apply: scale / shift must be 16-byte aligned");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  BnApplyDev p;
  p.M = a->M; p.C = a->C; p.ldh = a->ldh; p.ldr = a->ldr; p.ldy = a->ldy;
  p.h = (const __nv_bfloat16*)a->h; p.scale = a->scale; p.shift = a->shift; p.act = a->act;
  p.residual = (const __nv_bfloat16*)a->residual; p.y = (__nv_bfloat16*)a->y;
  p.gate = a->gate; p.rows_per_sample = a->rows_per_sample > 0 ? a->rows_per_sample : 1;
  p.residual2 = (const __nv_bfloat16*)a->residual2; p.ldr2 = a->ldr2;
  const long long total = a->M * (a->C / 8);
  long long blocks = (total + 255) / 256;
  const long long cap = (long long)max_ctas() * 16;
  bn_apply_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "bn_apply: %s", cudaGetErrorString(e));
  return 0;
}

int bn_reduce_launch(const yamb_bn_reduce* a, cudaStream_t st) {
  if (!a || a->M <= 0 || a->C <= 0 || (a->C % 8) || !a->bn)
    return set_error(YAMB_EINVAL, "bn_reduce shape");
  int rc;
  if ((rc = check_bf16("bn_reduce", "dy", a->dy, a->lddy, a->C)) ||
      (rc = check_bf16("bn_reduce", "h", a->h, a->ldh, a->C)))
    return rc;
  if (a->z_scale && !a->z_shift) return set_error(YAMB_EINVAL, "bn_reduce: z_scale without z_shift");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  BnReduceDev p;
  p.M = a->M; p.C = a->C; p.lddy = a->lddy; p.ldh = a->ldh;
  p.dy = (const __nv_bfloat16*)a->dy; p.h = (const __nv_bfloat16*)a->h; p.bn = *a->bn;
  p.z_scale = a->z_scale; p.z_shift = a->z_scale ? a->z_shift : nullptr; p.z_act = a->z_act;
  const size_t smem = stats_smem(a->C);
  if ((rc = smem_optin("bn_reduce", (const void*)bn_reduce_kernel, smem))) return rc;
  const int CG = a->C / 8;
  const int PX = 256 / CG > 0 ? 256 / CG : 1;
  long long want = (a->M + PX - 1) / PX;
  int grid = (int)(want < (long long)2 * max_ctas() ? want : 2 * max_ctas());
  bn_reduce_kernel<<<grid, 256, smem, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "bn_reduce: %s", cudaGetErrorString(e));
  return 0;
}

int bn_stats_launch(const yamb_bn_stats* a, cudaStream_t st) {
  if (!a || a->M <= 0 || a->C <= 0 || (a->C % 8) || !a->bn)
    return set_error(YAMB_EINVAL, "bn_stats args");
  int rc;
  if ((rc = check_bf16("bn_stats", "h", a->h, a->ldh, a->C))) return rc;
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  BnStatsDev p;
  p.M = a->M; p.C = a->C; p.ldh = a->ldh;
  p.h = (const __nv_bfloat16*)a->h; p.bn = *a->bn;
  const size_t smem = stats_smem(a->C);
  if ((rc = smem_optin("bn_stats", (const void*)bn_stats_kernel, smem))) return rc;
  const int CG = a->C / 8;
  const int PX = 256 / CG > 0 ? 256 / CG : 1;
  long long want = (a->M + PX - 1) / PX;
  int grid = (int)(want < (long long)4 * max_ctas() ? want : 4 * max_ctas());
  bn_stats_kernel<<<grid, 256, smem, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "bn_stats: %s", cudaGetErrorString(e));
  return 0;
}

int bn_bwd_apply_launch(const yamb_bn_bwd_apply* a, cudaStream_t st) {
  if (!a || a->M <= 0 || a->C <= 0 || (a->C % 8) || !a->ca || !a->cb || !a->cc)
    return set_error(YAMB_EINVAL, "bn_bwd_apply args");
  int rc;
  if ((rc = check_bf16("bn_bwd_apply", "dy", a->dy, a->lddy, a->C)) ||
      (rc = check_bf16("bn_bwd_apply", "h", a->h, a->ldh, a->C)) ||
      (rc = check_bf16("bn_bwd_apply", "dh", a->dh, a->lddh, a->C)))
    return rc;
  if (a->z_scale && !a->z_shift)
    return set_error(YAMB_EINVAL, "bn_bwd_apply: z_scale without z_shift");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  BnBwdApplyDev p;
  p.M = a->M; p.C = a->C; p.lddy = a->lddy; p.ldh = a->ldh; p.lddh = a->lddh;
  p.dy = (const __nv_bfloat16*)a->dy; p.h = (const __nv_bfloat16*)a->h;
  p.z_scale = a->z_scale; p.z_shift = a->z_shift; p.z_act = a->z_act;
  p.ca = a->ca; p.cb = a->cb; p.cc = a->cc; p.dh = (__nv_bfloat16*)a->dh;
  const int CG = a->C / 8;
  const int PX = 256 / CG > 0 ? 256 / CG : 1;
  // one 4-row batch per pixel lane and CTA at least; up to 8 CTAs per SM (the SM's thread limit)
  long long want = (a->M + 4LL * PX - 1) / (4LL * PX);
  int grid = (int)(want < (long long)8 * max_ctas() ? want : 8 * max_ctas());
  bn_bwd_apply_kernel<<<grid, 256, 0, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "bn_bwd_apply: %s", cudaGetErrorString(e));
  return 0;
}

// pixel chunks per sample: enough CTAs to fill the GPU ~4x, every pixel lane with >= 4 rows
static int se_chunks(int N, int HW, int C) {
  const int PX = 256 / (C / 8) > 0 ? 256 / (C / 8) : 1;
  int want = (4 * max_ctas() + N - 1) / N;
  int most = HW / (4 * PX);
  if (most < 1) most = 1;
  if (want > most) want = most;
  return want < 1 ? 1 : want;
}

// Slabs of the [N][C] sums of se_rows_reduce, one per pixel chunk: a stream-ordered scratch when
// there are several (det_reduce stores their sum in chunk order afterwards), the output itself
// when there is one.  A thread owns one 8-channel group, so channels go in launches of 2048; the
// chunk count comes from the widest one and is the same for all.
static int se_slabs(int N, int HW, int C, float* out, cudaStream_t st, int* chunks, float** part) {
  *chunks = se_chunks(N, HW, C < 2048 ? C : 2048);
  *part = out;
  if (*chunks == 1) return 0;
  return det_alloc((size_t)*chunks * N * C * sizeof(float), st, part);
}

static int se_slabs_done(float* part, int chunks, int N, int C, float* out, cudaStream_t st,
                         const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    if (part != out) det_free(part, st);
    return set_error(YAMB_ECUDA, "%s: %s", what, cudaGetErrorString(e));
  }
  return part != out ? det_reduce_launch(part, chunks, (long long)N * C, out, st, false) : 0;
}

int se_pool_launch(const yamb_se_pool* a, cudaStream_t st) {
  if (!a || a->N <= 0 || a->HW <= 0 || a->C <= 0 || (a->C % 8))
    return set_error(YAMB_EINVAL, "se_pool shape");
  int rc;
  if ((rc = check_bf16("se_pool", "h", a->h, a->ldh, a->C))) return rc;
  if (a->N > 65535) return set_error(YAMB_EINVAL, "se_pool: N <= 65535");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  SePoolDev p;
  p.N = a->N; p.HW = a->HW; p.C = a->C; p.ldh = a->ldh;
  p.h = (const __nv_bfloat16*)a->h; p.scale = a->scale; p.shift = a->shift; p.act = a->act;
  int chunks;
  rc = se_slabs(a->N, a->HW, a->C, a->pooled, st, &chunks, &p.pooled);
  if (rc) return rc;
  p.out_ld = a->C;
  p.slab = (long long)a->N * a->C;
  for (int c0 = 0; c0 < a->C; c0 += 2048) {
    SePoolDev q = p;
    q.C = a->C - c0 < 2048 ? a->C - c0 : 2048;
    q.h = p.h + c0; q.scale = p.scale + c0; q.shift = p.shift + c0; q.pooled = p.pooled + c0;
    dim3 grid(chunks, a->N);
    se_pool_kernel<<<grid, 256, 0, st>>>(q);
  }
  return se_slabs_done(p.pooled, chunks, a->N, a->C, a->pooled, st, "se_pool");
}

int se_bwd_reduce_launch(const yamb_se_bwd_reduce* a, cudaStream_t st) {
  if (!a || a->N <= 0 || a->HW <= 0 || a->C <= 0 || (a->C % 8))
    return set_error(YAMB_EINVAL, "se_bwd_reduce shape");
  int rc;
  if ((rc = check_bf16("se_bwd_reduce", "dy", a->dy, a->ldd, a->C)) ||
      (rc = check_bf16("se_bwd_reduce", "h", a->h, a->ldh, a->C)))
    return rc;
  if (a->N > 65535) return set_error(YAMB_EINVAL, "se_bwd_reduce: N <= 65535");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  SeBwdReduceDev p;
  p.N = a->N; p.HW = a->HW; p.C = a->C; p.ldd = a->ldd; p.ldh = a->ldh;
  p.dy = (const __nv_bfloat16*)a->dy; p.h = (const __nv_bfloat16*)a->h;
  p.scale = a->scale; p.shift = a->shift; p.act = a->act;
  int chunks;
  rc = se_slabs(a->N, a->HW, a->C, a->dgate, st, &chunks, &p.dgate);
  if (rc) return rc;
  p.out_ld = a->C;
  p.slab = (long long)a->N * a->C;
  for (int c0 = 0; c0 < a->C; c0 += 2048) {
    SeBwdReduceDev q = p;
    q.C = a->C - c0 < 2048 ? a->C - c0 : 2048;
    q.h = p.h + c0; q.dy = p.dy + c0; q.scale = p.scale + c0; q.shift = p.shift + c0;
    q.dgate = p.dgate + c0;
    dim3 grid(chunks, a->N);
    se_bwd_reduce_kernel<<<grid, 256, 0, st>>>(q);
  }
  return se_slabs_done(p.dgate, chunks, a->N, a->C, a->dgate, st, "se_bwd_reduce");
}

int se_bwd_apply_launch(const yamb_se_bwd_apply* a, cudaStream_t st) {
  if (!a || a->M <= 0 || a->C <= 0 || (a->C % 8) || !a->bn || a->rows_per_sample <= 0)
    return set_error(YAMB_EINVAL, "se_bwd_apply shape");
  int rc;
  if ((rc = check_bf16("se_bwd_apply", "dy", a->dy, a->ldd, a->C)) ||
      (rc = check_bf16("se_bwd_apply", "h", a->h, a->ldh, a->C)) ||
      (rc = check_bf16("se_bwd_apply", "dz", a->dz, a->ldz, a->C)))
    return rc;
  const int ldg = a->ldg > 0 ? a->ldg : a->C;
  if (!a->gate || !a->dpool ||
      ((reinterpret_cast<uintptr_t>(a->gate) | reinterpret_cast<uintptr_t>(a->dpool)) & 15) ||
      (ldg % 4))
    return set_error(YAMB_EINVAL, "se_bwd_apply: gate / dpool must be 16-byte aligned, pitch % 4 == 0");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  SeBwdApplyDev p;
  p.M = a->M; p.C = a->C; p.ldd = a->ldd; p.ldh = a->ldh; p.ldz = a->ldz;
  p.rows_per_sample = a->rows_per_sample;
  p.dy = (const __nv_bfloat16*)a->dy; p.h = (const __nv_bfloat16*)a->h;
  p.scale = a->scale; p.shift = a->shift; p.act = a->act;
  p.gate = a->gate; p.dpool = a->dpool; p.ldg = ldg;
  p.dz = (__nv_bfloat16*)a->dz; p.bn = *a->bn;
  const size_t smem = stats_smem(a->C);
  if ((rc = smem_optin("se_bwd_apply", (const void*)se_bwd_apply_kernel, smem))) return rc;
  const int CG = a->C / 8;
  const int PX = 256 / CG > 0 ? 256 / CG : 1;
  long long want = (a->M + PX - 1) / PX;
  int grid = (int)(want < (long long)2 * max_ctas() ? want : 2 * max_ctas());
  se_bwd_apply_kernel<<<grid, 256, smem, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "se_bwd_apply: %s", cudaGetErrorString(e));
  return 0;
}

int se_bwd_stats_launch(const yamb_se_bwd_stats* a, cudaStream_t st) {
  if (!a || a->N <= 0 || a->HW <= 0 || a->C <= 0 || (a->C % 8))
    return set_error(YAMB_EINVAL, "se_bwd_stats shape");
  int rc;
  if ((rc = check_bf16("se_bwd_stats", "dy", a->dy, a->ldd, a->C)) ||
      (rc = check_bf16("se_bwd_stats", "h", a->h, a->ldh, a->C)))
    return rc;
  if (!a->scale || !a->shift || !a->mean || !a->invstd || !a->dgate || !a->sums)
    return set_error(YAMB_EINVAL, "se_bwd_stats: null pointer");
  if (a->act < YAMB_ACT_NONE || a->act > YAMB_ACT_HSWISH)
    return set_error(YAMB_EINVAL, "se_bwd_stats: act=%d", a->act);
  if (a->N > 65535) return set_error(YAMB_EINVAL, "se_bwd_stats: N <= 65535");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  // the launch plan and dgate slabs of se_bwd_reduce_launch
  SeBwdStatsDev p;
  p.r.N = a->N; p.r.HW = a->HW; p.r.C = a->C; p.r.ldd = a->ldd; p.r.ldh = a->ldh;
  p.r.dy = (const __nv_bfloat16*)a->dy; p.r.h = (const __nv_bfloat16*)a->h;
  p.r.scale = a->scale; p.r.shift = a->shift; p.r.act = a->act;
  int chunks;
  rc = se_slabs(a->N, a->HW, a->C, a->dgate, st, &chunks, &p.r.dgate);
  if (rc) return rc;
  p.r.out_ld = a->C;
  p.r.slab = (long long)a->N * a->C;
  p.st.mean = a->mean; p.st.invstd = a->invstd;
  p.st.plane = (long long)a->N * a->C;
  const long long nsum = 4 * p.st.plane;
  p.st.sums = a->sums;
  if (chunks > 1) {
    float* part = nullptr;
    if ((rc = det_alloc((size_t)chunks * nsum * sizeof(double), st, &part))) {
      if (p.r.dgate != a->dgate) det_free(p.r.dgate, st);
      return rc;
    }
    p.st.sums = reinterpret_cast<double*>(part);
  }
  for (int c0 = 0; c0 < a->C; c0 += 2048) {
    SeBwdStatsDev q = p;
    q.r.C = a->C - c0 < 2048 ? a->C - c0 : 2048;
    q.r.h = p.r.h + c0; q.r.dy = p.r.dy + c0; q.r.scale = p.r.scale + c0; q.r.shift = p.r.shift + c0;
    q.r.dgate = p.r.dgate + c0;
    q.st.mean = p.st.mean + c0; q.st.invstd = p.st.invstd + c0; q.st.sums = p.st.sums + c0;
    dim3 grid(chunks, a->N);
    se_bwd_stats_kernel<<<grid, 256, 0, st>>>(q);
  }
  if (chunks > 1) {
    const long long blocks = (nsum + 255) / 256, cap = 4LL * max_ctas();
    se_sums_reduce_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>(p.st.sums, chunks, nsum,
                                                                               a->sums);
    det_free(reinterpret_cast<float*>(p.st.sums), st);
  }
  return se_slabs_done(p.r.dgate, chunks, a->N, a->C, a->dgate, st, "se_bwd_stats");
}

int se_bn_bwd_finalize_launch(const yamb_se_bn_bwd_finalize_args* a, cudaStream_t st) {
  if (!a || a->N <= 0 || a->C <= 0 || !a->bn) return set_error(YAMB_EINVAL, "se_bn_bwd_finalize shape");
  if (a->lds < a->C || a->ldg < a->C)
    return set_error(YAMB_EINVAL, "se_bn_bwd_finalize: lds=%d ldg=%d need >= C=%d", a->lds, a->ldg, a->C);
  const yamb_bn_bwd& b = *a->bn;
  if (!a->sums || !a->gate || !a->dpool || !b.mean || !b.invstd || !b.ca || !b.cb || !b.cc)
    return set_error(YAMB_EINVAL, "se_bn_bwd_finalize: null pointer");
  if (b.count <= 0) return set_error(YAMB_EINVAL, "se_bn_bwd_finalize: bn count %lld", (long long)b.count);
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  SeBnFinalizeDev p;
  p.N = a->N; p.C = a->C; p.lds = a->lds; p.ldg = a->ldg;
  p.sums = a->sums; p.gate = a->gate; p.dpool = a->dpool; p.bn = b;
  se_bn_bwd_finalize_kernel<<<(a->C + 31) / 32, 256, 0, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "se_bn_bwd_finalize: %s", cudaGetErrorString(e));
  return 0;
}

}  // namespace yamb
