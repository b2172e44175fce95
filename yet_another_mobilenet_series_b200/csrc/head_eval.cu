// Eval-mode head of the network in one launch, sm_90a: the 1x1 ConvBNReLU (reference
// models/mobilenet_supernet.py:152-158) followed by the full-extent AvgPool2d (:159), with the
// BatchNorm folded from its running statistics:
//
//   pooled[n][c] = bf16( (1/HW) * sum_p bf16(act(scale[c] * bf16(x[n,p,:] . W[c,:]) + shift[c])) )
//
// The rounding points of the unfused sequence (head GEMM -> bn_apply -> mean) are kept; only the
// order of the mean's sum differs, and it is fixed: per 64-pixel chunk, the two rows of a thread,
// then a butterfly over the 8 lanes sharing a column, then the four warps in order, then the
// chunks in order — the same bits on every run, no atomics.  Neither the conv output h nor the
// activation a is written to HBM.
//
// CTA = one warpgroup = (image n, 64 output channels).  The CTA's weight rows [64][Cin] and the
// image's pixels [64][Cin] (one m64 chunk; images with HW > 64 loop over chunks) are staged in
// shared memory as 128-byte-swizzled K-major panels of 64 channels (cp.async, zero-filled beyond
// HW / Cout / Cin) and multiplied by wgmma m64n64k16.  Cin <= 512: at most 128 KB of operands.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "host_util.h"
#include "prims.cuh"

namespace yamb {

constexpr int kHeadMaxCin = 512;

struct HeadDev {
  int N, HW, Cin, Cout, kpanels;
  const __nv_bfloat16* x;       // [N][HW][Cin]
  const __nv_bfloat16* w;       // [Cout][Cin]
  const float *scale, *shift;   // [Cout]
  int act;
  float inv_hw;
  __nv_bfloat16* pooled;        // [N][Cout]
};

// 64 rows x kpanels panels of 64 channels; row r of panel kb at kb*8192 + r*128, 16-byte chunk c
// of the row stored at chunk (c ^ (r & 7)) (the wgmma SWIZZLE_128B layout)
__device__ __forceinline__ void head_stage(uint8_t* dst, const __nv_bfloat16* src, int rows_valid,
                                           int Cin, int kpanels) {
  const int chunks = kpanels * 8;
  for (int e = threadIdx.x; e < 64 * chunks; e += 128) {
    const int r = e / chunks, q = e - r * chunks;
    const int kb = q >> 3, c = q & 7;
    const bool ok = r < rows_valid && q * 8 < Cin;
    const void* s = ok ? (const void*)(src + (size_t)r * Cin + q * 8) : (const void*)src;
    cp_async_zfill16(smem_u32(dst + kb * 8192 + r * 128 + ((c ^ (r & 7)) << 4)), s, ok ? 16 : 0);
  }
  cp_async_commit();
}

__global__ void __launch_bounds__(128) head_pool_eval_kernel(const __grid_constant__ HeadDev p) {
  extern __shared__ __align__(1024) unsigned char head_smem_raw[];
  // the swizzle pattern repeats every 1024 bytes: panels start on a 1024-byte boundary
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(head_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sB = smem;                                   // weights [64 channels][Cin]
  uint8_t* sA = smem + p.kpanels * 8192;                // pixels  [64][Cin]
  float* red = reinterpret_cast<float*>(sA + p.kpanels * 8192);   // [4 warps][64 columns]
  const int n = blockIdx.x, n0 = blockIdx.y * 64;
  const int tid = threadIdx.x, w = tid >> 5, l = tid & 31;
  head_stage(sB, p.w + (size_t)n0 * p.Cin, p.Cout - n0, p.Cin, p.kpanels);
  const ActParam ap = make_act(p.act);
  // per-thread (scale, shift) of the 16 columns it holds: col = 8j + 2(l%4) + e
  float sc[16], sh[16];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int c = n0 + 8 * j + 2 * (l & 3) + e;
      sc[2 * j + e] = c < p.Cout ? p.scale[c] : 0.f;
      sh[2 * j + e] = c < p.Cout ? p.shift[c] : 0.f;
    }
  const uint32_t sA_u = smem_u32(sA), sB_u = smem_u32(sB);
  const __nv_bfloat16* img = p.x + (size_t)n * p.HW * p.Cin;
  float total = 0.f;                                    // threads 0..63: column tid
  for (int p0 = 0; p0 < p.HW; p0 += 64) {
    const int rows = min(64, p.HW - p0);
    head_stage(sA, img + (size_t)p0 * p.Cin, rows, p.Cin, p.kpanels);
    cp_async_wait<0>();
    fence_proxy_async_smem();
    __syncthreads();
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    reg_fence(acc);
    wgmma_fence();
#pragma unroll 1
    for (int ks = 0; ks < 4 * p.kpanels; ++ks) {
      const uint32_t off = (uint32_t)((ks >> 2) * 8192 + (ks & 3) * 32);
      wgmma_m64n64<0, 0>(acc, gmma_smem_desc(sA_u + off, 16, 1024),
                         gmma_smem_desc(sB_u + off, 16, 1024), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(acc);
    // d[4j + 2h + e] -> row 16w + l/4 + 8h, column 8j + 2(l%4) + e
    const int r0 = 16 * w + (l >> 2);
    const bool v0 = r0 < rows, v1 = r0 + 8 < rows;
    float s[16];
    if (ap.kind == 0) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int i = 2 * j + e;
          const float a0 = round_bf16(fminf(fmaxf(fmaf(sc[i], round_bf16(acc[4 * j + e]), sh[i]), ap.lo), ap.hi));
          const float a1 = round_bf16(fminf(fmaxf(fmaf(sc[i], round_bf16(acc[4 * j + 2 + e]), sh[i]), ap.lo), ap.hi));
          s[i] = (v0 ? a0 : 0.f) + (v1 ? a1 : 0.f);
        }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int i = 2 * j + e;
          const float a0 = round_bf16(act_rt(fmaf(sc[i], round_bf16(acc[4 * j + e]), sh[i]), ap));
          const float a1 = round_bf16(act_rt(fmaf(sc[i], round_bf16(acc[4 * j + 2 + e]), sh[i]), ap));
          s[i] = (v0 ? a0 : 0.f) + (v1 ? a1 : 0.f);
        }
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      s[i] += __shfl_xor_sync(0xffffffffu, s[i], 4);
      s[i] += __shfl_xor_sync(0xffffffffu, s[i], 8);
      s[i] += __shfl_xor_sync(0xffffffffu, s[i], 16);
    }
    if (l < 4) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) red[w * 64 + 8 * j + 2 * l + e] = s[2 * j + e];
    }
    __syncthreads();                                    // red complete; sA free for the next chunk
    if (tid < 64) total += ((red[tid] + red[64 + tid]) + red[128 + tid]) + red[192 + tid];
    __syncthreads();
  }
  if (tid < 64 && n0 + tid < p.Cout)
    p.pooled[(size_t)n * p.Cout + n0 + tid] = __float2bfloat16_rn(total * p.inv_hw);
}

int head_pool_eval_launch(const yamb_head_pool_eval* a, cudaStream_t st) {
  if (!a || a->N <= 0 || a->HW <= 0 || !a->x || !a->w || !a->scale || !a->shift || !a->pooled)
    return set_error(YAMB_EINVAL, "head pool eval: bad arguments");
  if (a->Cin <= 0 || a->Cin % 8 || a->Cin > kHeadMaxCin || a->Cout <= 0 || a->Cout % 8)
    return set_error(YAMB_EINVAL, "head pool eval: Cin=%d (multiple of 8, <= %d), Cout=%d "
                     "(multiple of 8) not covered", a->Cin, kHeadMaxCin, a->Cout);
  if (a->act < YAMB_ACT_NONE || a->act > YAMB_ACT_HSWISH)
    return set_error(YAMB_EINVAL, "head pool eval: act=%d", a->act);
  if ((reinterpret_cast<uintptr_t>(a->x) | reinterpret_cast<uintptr_t>(a->w)) & 15)
    return set_error(YAMB_EINVAL, "head pool eval: x / w must be 16-byte aligned");
  if ((long long)a->N * a->HW >= (1LL << 31) || (a->Cout + 63) / 64 > 65535)
    return set_error(YAMB_EINVAL, "head pool eval: too large");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  HeadDev p;
  p.N = a->N; p.HW = a->HW; p.Cin = a->Cin; p.Cout = a->Cout;
  p.kpanels = (a->Cin + 63) / 64;
  p.x = (const __nv_bfloat16*)a->x; p.w = (const __nv_bfloat16*)a->w;
  p.scale = a->scale; p.shift = a->shift; p.act = a->act;
  p.inv_hw = 1.f / (float)a->HW;
  p.pooled = (__nv_bfloat16*)a->pooled;
  const size_t smem = 1024 + (size_t)2 * p.kpanels * 8192 + 4 * 64 * sizeof(float);
  const int rc = smem_optin("head pool eval", (const void*)head_pool_eval_kernel, smem);
  if (rc) return rc;
  head_pool_eval_kernel<<<dim3(a->N, (a->Cout + 63) / 64), 128, smem, st>>>(p);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "head pool eval: %s", cudaGetErrorString(e));
  return 0;
}

}  // namespace yamb
