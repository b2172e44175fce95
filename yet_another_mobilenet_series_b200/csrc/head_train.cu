// Training-mode head of the network after its 1x1 convolution, sm_90a: BatchNorm with the batch
// statistics the head GEMM's epilogue took, the activation, and the full-extent AvgPool2d
// (reference models/mobilenet_supernet.py:152-159), with neither the activation a nor its
// broadcast gradient in HBM:
//
//   forward : pooled[n][c] = bf16((1/HW) * sum_p bf16(act(scale[c] * h[n,p,c] + shift[c])))
//   backward: dz = act'(scale*h + shift) * dpooled[n][c] * (1/HW)
//             reduce: sum(dz), sum(dz * xhat) -> bn_bwd_finalize (dgamma, dbeta, ca, cb, cc)
//             apply : dh = bf16(ca*dz + cb*h + cc)
//
// The rounding points of a are those of bn_apply (fmaf, activation, RN to bf16), so only the
// order of the pool's sum differs from the unfused sequence; it is fixed (per-thread pixel lanes,
// the lanes in order, the pixel-chunk slabs in order) and has no atomics.  The backward passes
// have the thread layout and arithmetic of bn_reduce / bn_bwd_apply (csrc/elementwise.cu) with
// dy = dpooled[n][c] / HW taken from the [N][C] gradient instead of a [pixels][C] tensor.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "bn_finalize.cuh"
#include "host_util.h"
#include "prims.cuh"

namespace yamb {

// A thread owns one 8-channel group cg and a pixel lane px (tid = px * CGw + cg - cgb); channel
// groups beyond 256 are covered by looping cgb, as in bn_reduce.
struct Lanes {
  int CG, CGw, PX;
  __device__ __forceinline__ explicit Lanes(int C) {
    CG = C / 8;
    CGw = CG >= 256 ? 256 : CG;
    PX = 256 / CGw;
  }
  __device__ __forceinline__ int cg(int cgb) const { return cgb + (int)threadIdx.x % CGw; }
  __device__ __forceinline__ int px() const { return (int)threadIdx.x / CGw; }
};

__device__ __forceinline__ void load8(const float* p, float (&v)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

struct HeadTrainFwdDev {
  int N, HW, C;
  const __nv_bfloat16* h;
  const float *scale, *shift;
  int act;
  float inv_hw;
  float* slab;            // [gridDim.x][N][C] per-chunk sums, or nullptr: one chunk, write pooled
  __nv_bfloat16* pooled;  // [N][C]
};

// grid (pixel chunks, N): CTA (k, n) sums the pixels [k*rows_per, (k+1)*rows_per) of image n, with
// 4 rows in flight per thread
__global__ void __launch_bounds__(256) head_pool_train_fwd_kernel(const __grid_constant__ HeadTrainFwdDev p) {
  __shared__ float red[256][9];
  const Lanes L(p.C);
  const int n = blockIdx.y;
  const int rows_per = (p.HW + gridDim.x - 1) / gridDim.x;
  const int r0 = blockIdx.x * rows_per, r1 = min(p.HW, r0 + rows_per);
  const ActParam ap = make_act(p.act);
  for (int cgb = 0; cgb < L.CG; cgb += 256) {
    const int cg = L.cg(cgb), px = L.px();
    const bool active = cg < L.CG && px < L.PX;
    float s[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) s[e] = 0.f;
    if (active) {
      const int c0 = cg * 8;
      float sc[8], sh[8];
      load8(p.scale + c0, sc);
      load8(p.shift + c0, sh);
      const __nv_bfloat16* hb = p.h + (size_t)n * p.HW * p.C + c0;
      auto body = [&](const uint4& u) {
        float v[8];
        unpack8(u, v);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = fmaf(sc[e], v[e], sh[e]);
        act_vec<8>(v, ap);
#pragma unroll
        for (int e = 0; e < 8; ++e) s[e] += round_bf16(v[e]);
      };
      int i = r0 + px;
      for (; i + 3 * L.PX < r1; i += 4 * L.PX) {
        uint4 u[4];
#pragma unroll
        for (int j = 0; j < 4; ++j)
          u[j] = __ldg(reinterpret_cast<const uint4*>(hb + (size_t)(i + j * L.PX) * p.C));
#pragma unroll
        for (int j = 0; j < 4; ++j) body(u[j]);
      }
      for (; i < r1; i += L.PX) body(__ldg(reinterpret_cast<const uint4*>(hb + (size_t)i * p.C)));
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) red[threadIdx.x][e] = s[e];
    __syncthreads();
    if (active && px == 0) {
      const size_t o = (size_t)n * p.C + cg * 8;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        float t = 0.f;
        for (int j = 0; j < L.PX; ++j) t += red[threadIdx.x + j * L.CGw][e];
        if (p.slab)
          p.slab[(size_t)blockIdx.x * p.N * p.C + o + e] = t;
        else
          p.pooled[o + e] = __float2bfloat16_rn(t * p.inv_hw);
      }
    }
    __syncthreads();
  }
}

// pooled[i] = bf16((sum over k in order of slab[k][i]) * inv_hw)
__global__ void __launch_bounds__(256) head_pool_train_finish_kernel(const float* __restrict__ slab, int nslab,
                                                                     long long n, float inv_hw,
                                                                     __nv_bfloat16* __restrict__ pooled) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    float t = 0.f;
    for (int k = 0; k < nslab; ++k) t += slab[(size_t)k * n + i];
    pooled[i] = __float2bfloat16_rn(t * inv_hw);
  }
}

struct HeadTrainBwdDev {
  long long M;
  int HW, C;
  const __nv_bfloat16* h;
  const float *scale, *shift;
  int act;
  const __nv_bfloat16* dpooled;
  float inv_hw;
  yamb_bn_bwd bn;
  __nv_bfloat16* dh;
};

// dz of one row of 8 channels: dy = dpooled[row / HW][c0..] / HW, times act'(z), z = zs*h + zt
__device__ __forceinline__ void head_dz(const HeadTrainBwdDev& p, long long row, int c0,
                                        const float (&hv)[8], const float (&zs)[8],
                                        const float (&zt)[8], const ActParam& zap, float (&d)[8]) {
  const unsigned n = (unsigned)row / (unsigned)p.HW;        // M < 2^31 (launcher)
  unpack8(__ldg(reinterpret_cast<const uint4*>(p.dpooled + (size_t)n * p.C + c0)), d);
  float z[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    d[e] *= p.inv_hw;
    z[e] = fmaf(zs[e], hv[e], zt[e]);
  }
  act_bwd_vec<8>(d, z, zap, p.act);
}

// pass 1: sum(dz), sum(dz * xhat) per channel + BatchNorm-backward finalize (last CTA)
__global__ void __launch_bounds__(256) head_pool_train_reduce_kernel(const __grid_constant__ HeadTrainBwdDev p) {
  extern __shared__ stat_t s_part[];  // [2][C], double
  const Lanes L(p.C);
  for (int i = threadIdx.x; i < 2 * p.C; i += blockDim.x) s_part[i] = 0.0;
  __syncthreads();
  const ActParam zap = make_act(p.act);
  for (int cgb = 0; cgb < L.CG; cgb += 256) {
    const int cg = L.cg(cgb), px = L.px();
    const bool active = cg < L.CG && px < L.PX;
    float s[8], q[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) s[e] = q[e] = 0.f;
    if (active) {
      const int c0 = cg * 8;
      float mu[8], rs[8], zs[8], zt[8];
      load8(p.bn.mean + c0, mu);
      load8(p.bn.invstd + c0, rs);
      load8(p.scale + c0, zs);
      load8(p.shift + c0, zt);
      const long long rstep = (long long)gridDim.x * L.PX;
      for (long long row = (long long)blockIdx.x * L.PX + px; row < p.M; row += 4 * rstep) {
        uint4 uh[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const long long r2 = row + j * rstep;
          uh[j] = r2 < p.M ? __ldg(reinterpret_cast<const uint4*>(p.h + r2 * p.C + c0))
                           : make_uint4(0u, 0u, 0u, 0u);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const long long r2 = row + j * rstep;
          if (r2 >= p.M) break;
          float hv[8], d[8];
          unpack8(uh[j], hv);
          head_dz(p, r2, c0, hv, zs, zt, zap, d);
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            s[e] += d[e];
            q[e] = fmaf(d[e], (hv[e] - mu[e]) * rs[e], q[e]);
          }
        }
      }
    }
    cta_stats_merge(s_part, p.C, L.CGw, L.PX, cg, px, active, s, q);
  }
  __syncthreads();
  if (publish_partials(s_part, p.C, p.bn.partials, p.bn.counter)) {
    bn_bwd_finalize(p.bn, p.C);
    __syncthreads();
    if (threadIdx.x == 0) *p.bn.counter = 0;
  }
}

// pass 2: dh = ca*dz + cb*h + cc, the arithmetic of bn_bwd_apply (RN to bf16)
__global__ void __launch_bounds__(256) head_pool_train_apply_kernel(const __grid_constant__ HeadTrainBwdDev p) {
  const Lanes L(p.C);
  const ActParam zap = make_act(p.act);
  for (int cgb = 0; cgb < L.CG; cgb += 256) {
    const int cg = L.cg(cgb), px = L.px();
    if (cg >= L.CG || px >= L.PX) continue;
    const int c0 = cg * 8;
    float ca[8], cb[8], cc[8], zs[8], zt[8];
    load8(p.bn.ca + c0, ca);
    load8(p.bn.cb + c0, cb);
    load8(p.bn.cc + c0, cc);
    load8(p.scale + c0, zs);
    load8(p.shift + c0, zt);
    const long long rstep = (long long)gridDim.x * L.PX;
    for (long long row = (long long)blockIdx.x * L.PX + px; row < p.M; row += 4 * rstep) {
      uint4 uh[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const long long r2 = row + j * rstep;
        uh[j] = r2 < p.M ? __ldg(reinterpret_cast<const uint4*>(p.h + r2 * p.C + c0))
                         : make_uint4(0u, 0u, 0u, 0u);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const long long r2 = row + j * rstep;
        if (r2 >= p.M) break;
        float hv[8], d[8];
        unpack8(uh[j], hv);
        head_dz(p, r2, c0, hv, zs, zt, zap, d);
#pragma unroll
        for (int e = 0; e < 8; ++e) d[e] = fmaf(ca[e], d[e], fmaf(cb[e], hv[e], cc[e]));
        *reinterpret_cast<uint4*>(p.dh + r2 * p.C + c0) = pack8(d);
      }
    }
  }
}

// ---- launchers -----------------------------------------------------------------------------------
static bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

static int check_shape(const char* fn, int N, int HW, int C, const void* h, const float* scale,
                       const float* shift, int act) {
  if (N <= 0 || HW <= 0 || C <= 0 || C % 8)
    return set_error(YAMB_EINVAL, "%s: N=%d HW=%d C=%d (C a positive multiple of 8)", fn, N, HW, C);
  if ((long long)N * HW >= (1LL << 31) || N > 65535)
    return set_error(YAMB_EINVAL, "%s: too large (N*HW < 2^31, N <= 65535)", fn);
  if (!h || !scale || !shift || misaligned16(h) || misaligned16(scale) || misaligned16(shift))
    return set_error(YAMB_EINVAL, "%s: h / scale / shift missing or not 16-byte aligned", fn);
  if (act < YAMB_ACT_NONE || act > YAMB_ACT_HSWISH) return set_error(YAMB_EINVAL, "%s: act=%d", fn, act);
  return 0;
}

static int pixel_lanes(int C) { return C / 8 >= 256 ? 1 : 256 / (C / 8); }

int head_pool_train_fwd_launch(const yamb_head_pool_train* a, cudaStream_t st) {
  if (!a) return set_error(YAMB_EINVAL, "head pool train fwd: NULL arguments");
  int rc = check_shape("head pool train fwd", a->N, a->HW, a->C, a->h, a->scale, a->shift, a->act);
  if (rc) return rc;
  if (!a->pooled) return set_error(YAMB_EINVAL, "head pool train fwd: pooled is NULL");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  HeadTrainFwdDev p;
  p.N = a->N; p.HW = a->HW; p.C = a->C;
  p.h = (const __nv_bfloat16*)a->h; p.scale = a->scale; p.shift = a->shift; p.act = a->act;
  p.inv_hw = 1.f / (float)a->HW;
  p.pooled = (__nv_bfloat16*)a->pooled;
  p.slab = nullptr;
  // pixel chunks per image: enough CTAs to fill the GPU ~4x, every pixel lane with >= 4 rows
  int chunks = (4 * max_ctas() + a->N - 1) / a->N;
  const int most = a->HW / (4 * pixel_lanes(a->C));
  if (chunks > most) chunks = most;
  if (chunks < 1) chunks = 1;
  const long long n = (long long)a->N * a->C;
  if (chunks > 1 && (rc = det_alloc((size_t)chunks * n * sizeof(float), st, &p.slab))) return rc;
  head_pool_train_fwd_kernel<<<dim3(chunks, a->N), 256, 0, st>>>(p);
  if (chunks > 1) {
    const long long blocks = (n + 255) / 256, cap = 4LL * max_ctas();
    head_pool_train_finish_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>(
        p.slab, chunks, n, p.inv_hw, p.pooled);
  }
  const cudaError_t e = cudaGetLastError();
  if (chunks > 1) {
    const int rf = det_free(p.slab, st);
    if (e == cudaSuccess && rf) return rf;
  }
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "head pool train fwd: %s", cudaGetErrorString(e));
  return 0;
}

int head_pool_train_bwd_launch(const yamb_head_pool_train_grad* a, cudaStream_t st) {
  if (!a) return set_error(YAMB_EINVAL, "head pool train bwd: NULL arguments");
  int rc = check_shape("head pool train bwd", a->N, a->HW, a->C, a->h, a->scale, a->shift, a->act);
  if (rc) return rc;
  if (!a->dpooled || misaligned16(a->dpooled) || (a->dh && misaligned16(a->dh)))
    return set_error(YAMB_EINVAL, "head pool train bwd: dpooled missing, or dpooled / dh not 16-byte aligned");
  const yamb_bn_bwd& b = a->bn;
  if (!b.partials || !b.counter || !b.mean || !b.invstd || !b.ca || !b.cb || !b.cc ||
      misaligned16(b.mean) || misaligned16(b.invstd) || misaligned16(b.ca) || misaligned16(b.cb) ||
      misaligned16(b.cc))
    return set_error(YAMB_EINVAL, "head pool train bwd: bn needs partials, counter and 16-byte "
                     "aligned mean, invstd, ca, cb, cc");
  if (b.count != (long long)a->N * a->HW)
    return set_error(YAMB_EINVAL, "head pool train bwd: bn.count=%lld, N*HW=%lld", (long long)b.count,
                     (long long)a->N * a->HW);
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  HeadTrainBwdDev p;
  p.M = (long long)a->N * a->HW; p.HW = a->HW; p.C = a->C;
  p.h = (const __nv_bfloat16*)a->h; p.scale = a->scale; p.shift = a->shift; p.act = a->act;
  p.dpooled = (const __nv_bfloat16*)a->dpooled; p.inv_hw = 1.f / (float)a->HW;
  p.bn = b; p.dh = (__nv_bfloat16*)a->dh;
  const size_t smem = 2 * (size_t)a->C * sizeof(stat_t);
  if ((rc = smem_optin("head pool train reduce", (const void*)head_pool_train_reduce_kernel, smem)))
    return rc;
  const int PX = pixel_lanes(a->C);
  // grids of bn_reduce and bn_bwd_apply
  long long want = (p.M + PX - 1) / PX;
  int grid = (int)(want < 2LL * max_ctas() ? want : 2LL * max_ctas());
  head_pool_train_reduce_kernel<<<grid, 256, smem, st>>>(p);
  if (p.dh) {
    want = (p.M + 4LL * PX - 1) / (4LL * PX);
    grid = (int)(want < 8LL * max_ctas() ? want : 8LL * max_ctas());
    head_pool_train_apply_kernel<<<grid, 256, 0, st>>>(p);
  }
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "head pool train bwd: %s", cudaGetErrorString(e));
  return 0;
}

}  // namespace yamb
