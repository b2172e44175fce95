// Depthwise k x k convolution (k in {3,5,7}, stride 1/2) on NHWC bf16 activations, sm_90a.
//
// Replaces, behind yamb_depthwise_fwd / yamb_depthwise_bwd (include/yamb200.h), the
// nn.Conv2d(groups=C) + BatchNorm2d + activation library calls of the reference block
// (models/mobilenet_base.py:405-411 unfused, :275-281 fused) and their autograd backward.
//
// forward : y = dwconv(act(in_scale*x + in_shift))   — raw bf16 tiles (with halo) stream into
//           shared memory with cp.async (double-buffered); the producer's BatchNorm + activation
//           is applied ONCE per element, in place; per-channel sum / sum^2 of the bf16 output feed the next BatchNorm
//           (last-CTA finalize).
// backward: dh = ca*dz + cb*h + cc (BatchNorm backward of the depthwise output) is formed ONCE per
//           element while the gradient tile (with halo) is staged; da = dwconv^T(dh, w),
//           dwgt += sum dh * a (fused wgrad, accumulated in registers across the persistent loop),
//           dx = da * act'(z) with the statistics of the preceding BatchNorm's backward.
//
// (Kernel templates and launch helpers; instantiated by depthwise.cu — 32 / 64-channel tiles — and
// depthwise_narrow.cu — 8 / 16-channel tiles for the narrow branches of searched networks.)
//
// HBM-bound stencil: channels are the contiguous dimension; a thread owns 4 consecutive channels
// (8-byte global, 16-byte shared accesses); consecutive threads own consecutive channel groups and
// then consecutive pixels, so global accesses are contiguous runs of CT*2 bytes per pixel and
// shared accesses are bank-conflict free.  CTAs are persistent over (channel chunk, image tile).
#pragma once
#include <cuda_bf16.h>
#include <stdlib.h>
#include <cuda_runtime.h>

#include <mutex>

#include "bn_finalize.cuh"
#include "host_util.h"
#include "prims.cuh"

// resident CTAs per SM the 3x3 kernels are compiled for (register cap 64 Ki / (256 * n)); the
// profiling variant build overrides it (-DYAMB_DW_MINBLOCKS=3) to A/B occupancy against spills
#ifndef YAMB_DW_MINBLOCKS
#define YAMB_DW_MINBLOCKS 2
#endif

namespace yamb {

__device__ __forceinline__ void ld4(const __nv_bfloat16* p, float (&v)[4]) {
  const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
  v[0] = bf16lo(u.x); v[1] = bf16hi(u.x); v[2] = bf16lo(u.y); v[3] = bf16hi(u.y);
}
// round to bf16, store, and leave the rounded values in v
__device__ __forceinline__ void st4_round(__nv_bfloat16* p, float (&v)[4]) {
  const uint32_t a = pack_bf16(v[0], v[1]), b = pack_bf16(v[2], v[3]);
  v[0] = bf16lo(a); v[1] = bf16hi(a); v[2] = bf16lo(b); v[3] = bf16hi(b);
  *reinterpret_cast<uint2*>(p) = make_uint2(a, b);
}

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
struct DwFwdDev {
  int N, H, W, Ho, Wo, C, ldc;
  const __nv_bfloat16* x;
  const float* in_scale;
  const float* in_shift;
  int in_act;
  const float* w;
  __nv_bfloat16* y;
  int has_bn;
  yamb_bn_fwd bn;
  int tiles_h, tiles_w, chunks;
  int num_tiles;
};

// CT channels per tile (32 or 64); 256 threads = NCG channel groups x NSTRIP spatial threads, each
// computing TH x TW outputs of 4 channels from registers (every shared-memory load feeds up to
// K*K/S^2 FMAs: the stencil is bound by issue slots and shared-memory bandwidth, not by HBM).
template <int K, int S, int CT, int TW>
struct FwdGeom {
  static constexpr int TH = 4;                    // output rows per thread
  static constexpr int NCG = CT / 4;
  static constexpr int NSTRIP = 256 / NCG;
  static constexpr int TOW = 8 * TW;
  static constexpr int TOH = NSTRIP / 8 * TH;     // 8 (CT=64) or 16 (CT=32)
  static constexpr int IH = (TOH - 1) * S + K;
  static constexpr int IW = (TOW - 1) * S + K;
};

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// Forward, v4: the raw bf16 input tile (with halo) of tile t+1 streams into shared memory with
// cp.async (zero-fill outside the image) while tile t is transformed IN PLACE (BN + activation,
// rounded to bf16 like every other materialised activation) and convolved.
template <int K, int S, int CT, int TW>
__global__ void __launch_bounds__(256, (K == 3 ? YAMB_DW_MINBLOCKS : 1)) dw_fwd_kernel(
    const __grid_constant__ DwFwdDev p) {
  using G = FwdGeom<K, S, CT, TW>;
  constexpr int P = (K - 1) / 2;
  constexpr int TH = G::TH, NCG = G::NCG, IH = G::IH, IW = G::IW;
  constexpr int IR = (TH - 1) * S + K;     // input rows one thread reads
  constexpr int IC = (TW - 1) * S + K;     // input columns one thread reads
  constexpr int V8 = CT / 8;               // 16-byte vectors per pixel
  constexpr int PSTEP = 256 / V8;          // pixels one pass of the CTA covers
  constexpr int NPIX = IH * IW;
  constexpr int TILE_ELEMS = NPIX * CT;    // bf16 elements per staging buffer
  extern __shared__ __align__(16) float smem_f[];
  __nv_bfloat16* s_raw = reinterpret_cast<__nv_bfloat16*>(smem_f);  // [2][TILE_ELEMS]
  stat_t* s_part = reinterpret_cast<stat_t*>(smem_f + TILE_ELEMS);  // [2][CT] statistics of the current chunk (double)
  const int tid = threadIdx.x;
  for (int i = tid; i < 2 * CT; i += 256) s_part[i] = 0.0;
  const ActParam ap = make_act(p.in_scale ? p.in_act : ACT_NONE);
  const bool identity = p.in_scale == nullptr;
  const int cg = tid % NCG;
  const int strip = tid / NCG;
  const int sx = strip % 8, sy = strip / 8;
  const int g8 = tid % V8, pslot = tid / V8;   // staging / transform role: fixed 8-channel group
  float2 wreg[K * K][2];
  float sc8[8], sh8[8];
  float ssum[4] = {0.f, 0.f, 0.f, 0.f}, ssq[4] = {0.f, 0.f, 0.f, 0.f};
  int cur_chunk = -1;
  const unsigned tiles_per_img = (unsigned)(p.tiles_h * p.tiles_w);
  const unsigned tiles_per_chunk = (unsigned)p.N * tiles_per_img;

  // tile coordinates advance incrementally (tiles of a CTA are consecutive): one division-based
  // decode per CTA instead of three software divisions per tile
  struct Coord { int chunk, n, ty, tx; };
  auto decode = [&](unsigned t) {
    Coord c;
    c.chunk = (int)(t / tiles_per_chunk);
    unsigned r = t - (unsigned)c.chunk * tiles_per_chunk;
    c.n = (int)(r / tiles_per_img);
    r -= (unsigned)c.n * tiles_per_img;
    c.ty = (int)(r / (unsigned)p.tiles_w);
    c.tx = (int)(r - (unsigned)c.ty * p.tiles_w);
    return c;
  };
  auto advance = [&](Coord c) {
    if (++c.tx == p.tiles_w) {
      c.tx = 0;
      if (++c.ty == p.tiles_h) {
        c.ty = 0;
        if (++c.n == p.N) { c.n = 0; ++c.chunk; }
      }
    }
    return c;
  };
  constexpr int ITER = (NPIX + PSTEP - 1) / PSTEP;
  constexpr int DR = PSTEP / IW, DC = PSTEP % IW;
  const int pr0 = pslot / IW, pc0 = pslot % IW;   // this thread's first staged pixel
  // enqueue the cp.async copies of one tile into staging buffer `buf`; returns the bit mask of
  // the thread's in-image vectors (the transform pass of that tile reuses it)
  auto prefetch = [&](const Coord& tc, int buf) {
    const int iy0 = tc.ty * G::TOH * S - P, ix0 = tc.tx * G::TOW * S - P;
    const int c = tc.chunk * CT + g8 * 8;
    const bool cok = c < p.C;
    const __nv_bfloat16* img = p.x + (size_t)tc.n * p.H * p.W * p.ldc + c;
    const uint32_t dst = smem_u32(s_raw + buf * TILE_ELEMS + pslot * CT + g8 * 8);
    uint32_t mask = 0;
    int r = pr0, cc = pc0;
#pragma unroll
    for (int k = 0; k < ITER; ++k) {
      const int iy = iy0 + r, ix = ix0 + cc;
      bool ok = cok && (unsigned)iy < (unsigned)p.H && (unsigned)ix < (unsigned)p.W;
      if ((k + 1) * PSTEP > NPIX) ok = ok && (pslot + k * PSTEP < NPIX);
      const __nv_bfloat16* src = img + (ok ? (unsigned)((iy * p.W + ix) * p.ldc) : 0u);
      if ((k + 1) * PSTEP <= NPIX || pslot + k * PSTEP < NPIX)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + k * PSTEP * CT * 2),
                     "l"(src), "r"(ok ? 16 : 0)
                     : "memory");
      mask |= ok ? (1u << k) : 0u;
      cc += DC; r += DR;
      if (cc >= IW) { cc -= IW; ++r; }
    }
    return mask;
  };
  // per-chunk statistics: registers -> shared (once per chunk) -> one global reduction per channel
  auto flush_stats = [&](int chunk) {
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      float a = ssum[v], b = ssq[v];
      // lanes l, l + NCG, l + 2 NCG, ... of a warp own the same channels
#pragma unroll
      for (int off = NCG; off < 32; off <<= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, off);
        b += __shfl_xor_sync(0xffffffffu, b, off);
      }
      if ((tid & 31) < NCG) {
        atomicAdd(&s_part[cg * 4 + v], (stat_t)a);
        atomicAdd(&s_part[CT + cg * 4 + v], (stat_t)b);
      }
      ssum[v] = ssq[v] = 0.f;
    }
    __syncthreads();
    if (tid < 2 * CT) {
      const int c = chunk * CT + (tid % CT);
      const stat_t v = s_part[tid];
      if (c < p.C && v != 0.0) atomicAdd(p.bn.partials + (tid / CT) * p.C + c, v);
      s_part[tid] = 0.0;
    }
    __syncthreads();
  };

  // Each CTA walks a CONTIGUOUS range of tiles (row-major inside an image): the halo a tile
  // shares with its left / upper neighbours was fetched by the same SM a few tiles earlier and is
  // still in L2, instead of being requested by two SMs at the same instant.
  const unsigned t_end = (unsigned)(((unsigned long long)(blockIdx.x + 1) * p.num_tiles) / gridDim.x);
  unsigned t = (unsigned)(((unsigned long long)blockIdx.x * p.num_tiles) / gridDim.x);
  Coord cur = decode(t);
  uint32_t mask_next = 0;
  if (t < t_end) mask_next = prefetch(cur, 0);
  cp_async_commit();
  const uint32_t lo2 = pack_bf16(ap.lo, ap.lo), hi2 = pack_bf16(ap.hi, ap.hi);
  int buf = 0;
  for (; t < t_end; ++t, buf ^= 1) {
    const int chunk = cur.chunk, n = cur.n, ty = cur.ty, tx = cur.tx;
    const uint32_t mask = mask_next;
    const int cbase = chunk * CT;
    const int c0 = cbase + cg * 4;
    const bool cvalid = c0 < p.C;
    if (chunk != cur_chunk) {
      if (cur_chunk >= 0 && p.has_bn) flush_stats(cur_chunk);
      cur_chunk = chunk;
#pragma unroll
      for (int tp = 0; tp < K * K; ++tp) {
        float wv[4];
#pragma unroll
        for (int v = 0; v < 4; ++v)
          wv[v] = cvalid ? __ldg(p.w + (size_t)(c0 + v) * K * K + tp) : 0.f;
        wreg[tp][0] = make_float2(wv[0], wv[1]);
        wreg[tp][1] = make_float2(wv[2], wv[3]);
      }
      const int c8 = cbase + g8 * 8;
#pragma unroll
      for (int v = 0; v < 8; ++v) {
        const bool ok = !identity && c8 + v < p.C;
        sc8[v] = ok ? __ldg(p.in_scale + c8 + v) : 1.f;
        sh8[v] = ok ? __ldg(p.in_shift + c8 + v) : 0.f;
      }
    }
    const int oy0 = ty * G::TOH, ox0 = tx * G::TOW;
    __syncthreads();  // everyone is done computing from the buffer the next prefetch overwrites
    cur = advance(cur);
    if (t + 1 < t_end) mask_next = prefetch(cur, buf ^ 1);
    cp_async_commit();
    cp_async_wait<1>();  // this tile's copies (the older group) have landed
    __syncthreads();
    __nv_bfloat16* tile = s_raw + buf * TILE_ELEMS;
    // ---- in-place BN + activation (bf16 -> fp32 -> bf16); padding / halo stays exactly 0 ----
    if (!identity) {
      uint4* q0 = reinterpret_cast<uint4*>(tile + pslot * CT + g8 * 8);
#pragma unroll
      for (int k = 0; k < ITER; ++k) {
        if (mask & (1u << k)) {
          uint4* q = q0 + k * (PSTEP * CT / 8);
          const uint4 raw = *q;
          const uint32_t rw[4] = {raw.x, raw.y, raw.z, raw.w};
          uint32_t ow[4];
          if (ap.kind == 0) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float2 e = ffma2(make_float2(sc8[2 * j], sc8[2 * j + 1]),
                                     make_float2(bf16lo(rw[j]), bf16hi(rw[j])),
                                     make_float2(sh8[2 * j], sh8[2 * j + 1]));
              ow[j] = clamp_bf16x2(pack_bf16(e.x, e.y), lo2, hi2);
            }
          } else {
            float e8[8];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              e8[2 * j] = fmaf(sc8[2 * j], bf16lo(rw[j]), sh8[2 * j]);
              e8[2 * j + 1] = fmaf(sc8[2 * j + 1], bf16hi(rw[j]), sh8[2 * j + 1]);
            }
            act_vec<8>(e8, ap);
#pragma unroll
            for (int j = 0; j < 4; ++j) ow[j] = pack_bf16(e8[2 * j], e8[2 * j + 1]);
          }
          *q = make_uint4(ow[0], ow[1], ow[2], ow[3]);
        }
      }
      __syncthreads();
    }
    // ---- stencil: TH x TW outputs x 4 channels per thread (packed fp32x2 FMAs) ----
    float2 acc2[TH][TW][2];
#pragma unroll
    for (int j = 0; j < TH; ++j)
#pragma unroll
      for (int i = 0; i < TW; ++i) acc2[j][i][0] = acc2[j][i][1] = make_float2(0.f, 0.f);
    const __nv_bfloat16* tbase = tile + ((sy * TH * S) * IW + sx * TW * S) * CT + cg * 4;
#pragma unroll
    for (int rr = 0; rr < IR; ++rr) {
#pragma unroll
      for (int cc = 0; cc < IC; ++cc) {
        const uint2 a = *reinterpret_cast<const uint2*>(tbase + (rr * IW + cc) * CT);
        const float2 alo = make_float2(bf16lo(a.x), bf16hi(a.x));
        const float2 ahi = make_float2(bf16lo(a.y), bf16hi(a.y));
#pragma unroll
        for (int j = 0; j < TH; ++j) {
          const int ky = rr - j * S;  // compile-time after unrolling
          if (ky >= 0 && ky < K) {
#pragma unroll
            for (int i = 0; i < TW; ++i) {
              const int kx = cc - i * S;
              if (kx >= 0 && kx < K) {
                acc2[j][i][0] = ffma2(wreg[ky * K + kx][0], alo, acc2[j][i][0]);
                acc2[j][i][1] = ffma2(wreg[ky * K + kx][1], ahi, acc2[j][i][1]);
              }
            }
          }
        }
      }
    }
    if (cvalid) {
      const int oyb = oy0 + sy * TH, oxb = ox0 + sx * TW;
      __nv_bfloat16* ybase = p.y + (size_t)n * p.Ho * p.Wo * p.ldc + c0 +
                             (unsigned)((oyb * p.Wo + oxb) * p.ldc);
      const unsigned rstride = (unsigned)(p.Wo * p.ldc);
#pragma unroll
      for (int j = 0; j < TH; ++j) {
#pragma unroll
        for (int i = 0; i < TW; ++i) {
          if (oyb + j < p.Ho && oxb + i < p.Wo) {
            const float2 lo = acc2[j][i][0], hi = acc2[j][i][1];
            *reinterpret_cast<uint2*>(ybase + j * rstride + i * p.ldc) =
                make_uint2(pack_bf16(lo.x, lo.y), pack_bf16(hi.x, hi.y));
            // statistics of the fp32 accumulators (the bf16 rounding of the stored value is
            // zero-mean noise of relative variance 2^-18/3: far below the parity tolerance)
            ssum[0] += lo.x; ssum[1] += lo.y; ssum[2] += hi.x; ssum[3] += hi.y;
            ssq[0] = fmaf(lo.x, lo.x, ssq[0]); ssq[1] = fmaf(lo.y, lo.y, ssq[1]);
            ssq[2] = fmaf(hi.x, hi.x, ssq[2]); ssq[3] = fmaf(hi.y, hi.y, ssq[3]);
          }
        }
      }
    }
  }
  cp_async_wait<0>();
  if (p.has_bn) {
    if (cur_chunk >= 0) flush_stats(cur_chunk);
    if (arrive_last(p.bn.counter)) {
      bn_fwd_finalize(p.bn, p.C);
      __syncthreads();
      if (threadIdx.x == 0) *p.bn.counter = 0;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------
struct DwBwdDev {
  int N, H, W, Ho, Wo, C, ldc;
  const __nv_bfloat16* dz;  // [N,Ho,Wo,ldc]
  const __nv_bfloat16* h;   // [N,Ho,Wo,ldc]
  const float *ca, *cb, *cc;
  const float* w;           // [C][K][K]
  float* dw;                // [C][K][K] +=
  float* part;              // [CTA][C][K][K] per-CTA weight-gradient partials (zero-filled)
  const __nv_bfloat16* x;   // [N,H,W,ldc] pre-BN input of the depthwise stage
  const float *in_scale, *in_shift;
  int in_act;
  __nv_bfloat16* dx;        // [N,H,W,ldc]
  const __nv_bfloat16* residual;
  int has_bn;
  yamb_bn_bwd bn;
  int tiles_h, tiles_w, chunks;
  int num_tiles;
};

// Input-space CTA tile TIH x TIW made of 2x2-pixel thread tiles (aligned to even coordinates, so
// with stride 2 every thread sees the same, compile-time parity pattern of the transposed
// convolution); the gradient region that touches it is RH x RW output pixels.
template <int K, int S, int CT>
struct BwdGeom {
  static constexpr int P = (K - 1) / 2;
  static constexpr int NCG = CT / 4;
  static constexpr int NSP = 256 / NCG;        // spatial threads: 16 (CT=64) or 32 (CT=32)
  static constexpr int TIW = 8;
  static constexpr int TIH = NSP / 4 * 2;      // 8 or 16
  static constexpr int RH = S == 1 ? TIH + K - 1 : (TIH + K - 1) / 2 + 1;
  static constexpr int RW = S == 1 ? TIW + K - 1 : (TIW + K - 1) / 2 + 1;
  static constexpr int R = S == 1 ? K + 1 : (K + 1) / 2;   // region rows/cols one thread tile reads
};

// Does tap index k (one axis) connect pixel offset a (0/1 inside the thread tile) with region
// offset r (relative to the thread tile's first region row)?  Compile-time after unrolling.
template <int K, int S>
__device__ __forceinline__ constexpr bool tap_hits(int a, int k, int r) {
  constexpr int P = (K - 1) / 2;
  if (S == 1) return a + 2 * P - k == r;
  const int d = a + P - k;
  if (d & 1) return false;
  return d / 2 + P / 2 == r;
}

// TAP0..TAP1: taps whose weight gradient this launch accumulates (all of them unless K == 7, where
// 49 x 4 accumulators do not fit the register file and a second, wgrad-only launch covers the rest).
// DGRAD: compute and store dx (+ statistics); false for that second launch.
//
// v4: the raw bf16 tiles of tile t+1 (dz and h over the gradient region, x over the input tile)
// stream into shared memory with cp.async while tile t is processed; dh = ca*dz + cb*h + cc is
// formed once per element, in place (bf16, like every other materialised gradient); a thread
// gathers a 2x2 pixel tile from registers: every staged gradient vector feeds up to 4 dgrad and
// 4 wgrad FMAs, all shared-memory offsets are immediates, no bounds or parity branches.
template <int K, int S, int CT, int TAP0, int TAP1, bool DGRAD>
__global__ void __launch_bounds__(256, (K == 3 ? YAMB_DW_MINBLOCKS : 1)) dw_bwd_kernel(
    const __grid_constant__ DwBwdDev p) {
  using G = BwdGeom<K, S, CT>;
  constexpr int P = G::P, TIH = G::TIH, TIW = G::TIW, RH = G::RH, RW = G::RW, R = G::R;
  constexpr int NCG = G::NCG;
  constexpr int NT = TAP1 - TAP0;
  constexpr int KK = K * K;
  constexpr int V8 = CT / 8;
  constexpr int PSTEP = 256 / V8;
  constexpr int NPR = RH * RW;              // pixels of the gradient region
  constexpr int NPX = TIH * TIW;            // pixels of the input tile
  constexpr int REG_ELEMS = NPR * CT;
  constexpr int X_ELEMS = NPX * CT;
  constexpr int BUF_ELEMS = 2 * REG_ELEMS + X_ELEMS;  // one staging buffer: dz | h | x
  extern __shared__ __align__(16) float smem_f[];
  __nv_bfloat16* s_raw = reinterpret_cast<__nv_bfloat16*>(smem_f);  // [2][BUF_ELEMS]
  float* s_tab = smem_f + BUF_ELEMS;         // [7][CT]: in_scale, in_shift, ca, cb, cc, mean, invstd
  float* s_w = s_tab + 7 * CT;               // [K*K][CT]
  float* s_gw = s_w + KK * CT;               // [K*K][CT]
  stat_t* s_part = reinterpret_cast<stat_t*>(s_gw + KK * CT);   // [2][CT], double
  const int tid = threadIdx.x;
  for (int i = tid; i < KK * CT; i += 256) s_gw[i] = 0.f;
  for (int i = tid; i < 2 * CT; i += 256) s_part[i] = 0.0;
  const int act = p.in_scale ? p.in_act : ACT_NONE;
  const ActParam ap = make_act(act);
  const int cg = tid % NCG;
  const int sp = tid / NCG;
  const int py = (sp / 4) * 2, px = (sp % 4) * 2;   // thread tile origin inside the CTA tile
  const int g8 = tid % V8, pslot = tid / V8;        // staging / transform role
  // first region row / column of the thread tile (see tap_hits)
  const int rr0 = S == 1 ? py : py / 2, rc0 = S == 1 ? px : px / 2;
  float2 gw[NT][2];
  float ssum[4] = {0.f, 0.f, 0.f, 0.f}, ssq[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int tp = 0; tp < NT; ++tp) gw[tp][0] = gw[tp][1] = make_float2(0.f, 0.f);
  int cur_chunk = -1;
  const unsigned tiles_per_img = (unsigned)(p.tiles_h * p.tiles_w);
  const unsigned tiles_per_chunk = (unsigned)p.N * tiles_per_img;

  // registers -> shared (per chunk) -> one global reduction per (tap, channel) / channel
  auto flush = [&](int chunk) {
    // the thread tiles that share a channel group add in a fixed order (deterministic sums)
    for (int g = 0; g < (256 + NCG - 1) / NCG; ++g) {
      if (sp == g) {
#pragma unroll
        for (int tp = 0; tp < NT; ++tp) {
          float* dst = &s_gw[(TAP0 + tp) * CT + cg * 4];
          dst[0] += gw[tp][0].x;
          dst[1] += gw[tp][0].y;
          dst[2] += gw[tp][1].x;
          dst[3] += gw[tp][1].y;
        }
      }
      __syncthreads();
    }
#pragma unroll
    for (int tp = 0; tp < NT; ++tp) gw[tp][0] = gw[tp][1] = make_float2(0.f, 0.f);
    if (DGRAD) {
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        atomicAdd(&s_part[cg * 4 + v], (stat_t)ssum[v]);
        atomicAdd(&s_part[CT + cg * 4 + v], (stat_t)ssq[v]);
        ssum[v] = ssq[v] = 0.f;
      }
    }
    __syncthreads();
    const int cbase = chunk * CT;
    for (int i = tid; i < KK * CT; i += 256) {
      const int tp = i / CT, c = cbase + i % CT;
      const float g = s_gw[i];
      if (c < p.C && g != 0.f) p.part[((size_t)blockIdx.x * p.C + c) * KK + tp] = g;   // once per CTA
      s_gw[i] = 0.f;
    }
    if (DGRAD && p.has_bn && tid < 2 * CT) {
      const int c = cbase + tid % CT;
      const stat_t v = s_part[tid];
      if (c < p.C && v != 0.0) atomicAdd(p.bn.partials + (tid / CT) * p.C + c, v);
      s_part[tid] = 0.0;
    }
    __syncthreads();
  };
  auto load_tables = [&](int chunk) {
    const int cbase = chunk * CT;
    for (int i = tid; i < CT; i += 256) {
      const int c = cbase + i;
      const bool ok = c < p.C;
      s_tab[i] = ok && p.in_scale ? __ldg(p.in_scale + c) : 1.f;
      s_tab[CT + i] = ok && p.in_scale ? __ldg(p.in_shift + c) : 0.f;
      s_tab[2 * CT + i] = ok ? __ldg(p.ca + c) : 0.f;
      s_tab[3 * CT + i] = ok ? __ldg(p.cb + c) : 0.f;
      s_tab[4 * CT + i] = ok ? __ldg(p.cc + c) : 0.f;
      s_tab[5 * CT + i] = ok && p.has_bn ? __ldg(p.bn.mean + c) : 0.f;
      s_tab[6 * CT + i] = ok && p.has_bn ? __ldg(p.bn.invstd + c) : 0.f;
    }
    for (int i = tid; i < KK * CT; i += 256) {
      const int tp = i / CT, c = cbase + i % CT;
      s_w[i] = c < p.C ? __ldg(p.w + (size_t)c * KK + tp) : 0.f;
    }
  };
  struct Coord { int chunk, n, ty, tx; };
  auto decode = [&](unsigned t) {
    Coord c;
    c.chunk = (int)(t / tiles_per_chunk);
    unsigned r = t - (unsigned)c.chunk * tiles_per_chunk;
    c.n = (int)(r / tiles_per_img);
    r -= (unsigned)c.n * tiles_per_img;
    c.ty = (int)(r / (unsigned)p.tiles_w);
    c.tx = (int)(r - (unsigned)c.ty * p.tiles_w);
    return c;
  };
  auto advance = [&](Coord c) {
    if (++c.tx == p.tiles_w) {
      c.tx = 0;
      if (++c.ty == p.tiles_h) {
        c.ty = 0;
        if (++c.n == p.N) { c.n = 0; ++c.chunk; }
      }
    }
    return c;
  };
  auto region_origin = [&](int ty, int tx, int& ry0, int& rx0) {
    const int y0 = ty * TIH, x0 = tx * TIW;
    ry0 = S == 1 ? y0 - P : (y0 - P + 1) >> 1;   // ceil((y0-P)/2), also right for < 0
    rx0 = S == 1 ? x0 - P : (x0 - P + 1) >> 1;
  };
  constexpr int ITER_R = (NPR + PSTEP - 1) / PSTEP, ITER_X = (NPX + PSTEP - 1) / PSTEP;
  constexpr int DR_R = PSTEP / RW, DC_R = PSTEP % RW;
  const int rr_first = pslot / RW, rc_first = pslot % RW;   // first staged region pixel
  const int xr_first = pslot / TIW, xc_first = pslot % TIW; // first staged input pixel (PSTEP % TIW == 0)
  // enqueue one tile's cp.async copies; returns the mask of this thread's in-image region vectors
  auto prefetch = [&](const Coord& tc, int buf) {
    int ry0, rx0;
    region_origin(tc.ty, tc.tx, ry0, rx0);
    const int c = tc.chunk * CT + g8 * 8;
    const bool cok = c < p.C;
    const uint32_t d_dz = smem_u32(s_raw + buf * BUF_ELEMS + pslot * CT + g8 * 8);
    const uint32_t d_h = d_dz + REG_ELEMS * 2, d_x = d_h + REG_ELEMS * 2;
    const size_t img_o = (size_t)tc.n * p.Ho * p.Wo * p.ldc + c;
    const __nv_bfloat16* gdz = p.dz + img_o;
    const __nv_bfloat16* gh = p.h + img_o;
    uint32_t mask = 0;
    int r = rr_first, cc = rc_first;
#pragma unroll
    for (int k = 0; k < ITER_R; ++k) {
      const int oy = ry0 + r, ox = rx0 + cc;
      bool ok = cok && (unsigned)oy < (unsigned)p.Ho && (unsigned)ox < (unsigned)p.Wo;
      if ((k + 1) * PSTEP > NPR) ok = ok && (pslot + k * PSTEP < NPR);
      const unsigned o = ok ? (unsigned)((oy * p.Wo + ox) * p.ldc) : 0u;
      if ((k + 1) * PSTEP <= NPR || pslot + k * PSTEP < NPR) {
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d_dz + k * PSTEP * CT * 2),
                     "l"(gdz + o), "r"(ok ? 16 : 0) : "memory");
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d_h + k * PSTEP * CT * 2),
                     "l"(gh + o), "r"(ok ? 16 : 0) : "memory");
      }
      mask |= ok ? (1u << k) : 0u;
      cc += DC_R; r += DR_R;
      if (cc >= RW) { cc -= RW; ++r; }
    }
    const __nv_bfloat16* gx = p.x + (size_t)tc.n * p.H * p.W * p.ldc + c;
    const int y0 = tc.ty * TIH, x0 = tc.tx * TIW;
#pragma unroll
    for (int k = 0; k < ITER_X; ++k) {
      const int y = y0 + xr_first + k * (PSTEP / TIW), x = x0 + xc_first;
      bool ok = cok && y < p.H && x < p.W;
      if ((k + 1) * PSTEP > NPX) ok = ok && (pslot + k * PSTEP < NPX);
      const unsigned o = ok ? (unsigned)((y * p.W + x) * p.ldc) : 0u;
      if ((k + 1) * PSTEP <= NPX || pslot + k * PSTEP < NPX)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d_x + k * PSTEP * CT * 2),
                     "l"(gx + o), "r"(ok ? 16 : 0) : "memory");
    }
    return mask;
  };

  // contiguous tile range per CTA (halo reuse in L2, see the forward kernel)
  const unsigned t_end = (unsigned)(((unsigned long long)(blockIdx.x + 1) * p.num_tiles) / gridDim.x);
  unsigned t = (unsigned)(((unsigned long long)blockIdx.x * p.num_tiles) / gridDim.x);
  Coord cur = decode(t);
  uint32_t mask_next = 0;
  __syncthreads();
  if (t < t_end) mask_next = prefetch(cur, 0);
  cp_async_commit();
  int buf = 0;
  for (; t < t_end; ++t, buf ^= 1) {
    const int chunk = cur.chunk, n = cur.n, ty = cur.ty, tx = cur.tx;
    const uint32_t mask = mask_next;
    const int cbase = chunk * CT;
    const int c0 = cbase + cg * 4;
    const bool cvalid = c0 < p.C;
    if (chunk != cur_chunk) {
      if (cur_chunk >= 0) flush(cur_chunk);
      cur_chunk = chunk;
      load_tables(chunk);
    }
    const int y0 = ty * TIH, x0 = tx * TIW;
    __syncthreads();  // previous tile's compute is done with the buffer the prefetch overwrites
    cur = advance(cur);
    if (t + 1 < t_end) mask_next = prefetch(cur, buf ^ 1);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    __nv_bfloat16* b_dz = s_raw + buf * BUF_ELEMS;
    const __nv_bfloat16* b_h = b_dz + REG_ELEMS;
    const __nv_bfloat16* b_x = b_h + REG_ELEMS;
    // ---- dh = ca*dz + cb*h + cc in place over the gradient region (0 outside the image) ----
    if (mask) {
      float2 ca2[4], cb2[4], cc2[4];
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        ca2[v] = *reinterpret_cast<const float2*>(s_tab + 2 * CT + g8 * 8 + 2 * v);
        cb2[v] = *reinterpret_cast<const float2*>(s_tab + 3 * CT + g8 * 8 + 2 * v);
        cc2[v] = *reinterpret_cast<const float2*>(s_tab + 4 * CT + g8 * 8 + 2 * v);
      }
      uint4* q0 = reinterpret_cast<uint4*>(b_dz + pslot * CT + g8 * 8);
#pragma unroll
      for (int k = 0; k < ITER_R; ++k) {
        if (mask & (1u << k)) {
          uint4* q = q0 + k * (PSTEP * CT / 8);
          const uint4 rdz = *q;
          const uint4 rh = *(q + REG_ELEMS / 8);
          const uint32_t wz[4] = {rdz.x, rdz.y, rdz.z, rdz.w}, wh[4] = {rh.x, rh.y, rh.z, rh.w};
          uint32_t ow[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 t1 = ffma2(cb2[j], make_float2(bf16lo(wh[j]), bf16hi(wh[j])), cc2[j]);
            const float2 d = ffma2(ca2[j], make_float2(bf16lo(wz[j]), bf16hi(wz[j])), t1);
            ow[j] = pack_bf16(d.x, d.y);
          }
          *q = make_uint4(ow[0], ow[1], ow[2], ow[3]);
        }
      }
    }
    __syncthreads();
    // ---- 2x2 input pixels per thread: dgrad gather + fused wgrad + act'/BN-backward epilogue ----
    const float4 sc = *reinterpret_cast<const float4*>(s_tab + cg * 4);
    const float4 sh = *reinterpret_cast<const float4*>(s_tab + CT + cg * 4);
    const __nv_bfloat16* xbase = b_x + (py * TIW + px) * CT + cg * 4;
    float2 a1p[2][2][2];
    bool valid[2][2];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        valid[a][b] = cvalid && (y0 + py + a) < p.H && (x0 + px + b) < p.W;
        const uint2 xr = *reinterpret_cast<const uint2*>(xbase + (a * TIW + b) * CT);
        float a1[4] = {fmaf(sc.x, bf16lo(xr.x), sh.x), fmaf(sc.y, bf16hi(xr.x), sh.y),
                       fmaf(sc.z, bf16lo(xr.y), sh.z), fmaf(sc.w, bf16hi(xr.y), sh.w)};
        act_vec<4>(a1, ap);
        if (p.in_scale) {  // the forward convolved the bf16-rounded activation
#pragma unroll
          for (int v = 0; v < 4; ++v) a1[v] = round_bf16(a1[v]);
        }
        if (!valid[a][b]) a1[0] = a1[1] = a1[2] = a1[3] = 0.f;   // zero padding of the forward
        a1p[a][b][0] = make_float2(a1[0], a1[1]);
        a1p[a][b][1] = make_float2(a1[2], a1[3]);
      }
    float2 da2[2][2][2];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 2; ++b) da2[a][b][0] = da2[a][b][1] = make_float2(0.f, 0.f);
    // The staged region is zero outside the image and covers every tap of every pixel of the
    // tile: no bounds tests; which (pixel, tap) pairs meet at a region offset is compile-time.
    const __nv_bfloat16* dbase = b_dz + (rr0 * RW + rc0) * CT + cg * 4;
#pragma unroll
    for (int r = 0; r < R; ++r) {
#pragma unroll
      for (int c = 0; c < R; ++c) {
        const uint2 dr = *reinterpret_cast<const uint2*>(dbase + (r * RW + c) * CT);
        const float2 dlo = make_float2(bf16lo(dr.x), bf16hi(dr.x));
        const float2 dhi = make_float2(bf16lo(dr.y), bf16hi(dr.y));
#pragma unroll
        for (int ky = 0; ky < K; ++ky) {
#pragma unroll
          for (int kx = 0; kx < K; ++kx) {
            const int tp = ky * K + kx;
#pragma unroll
            for (int a = 0; a < 2; ++a) {
#pragma unroll
              for (int b = 0; b < 2; ++b) {
                if (tap_hits<K, S>(a, ky, r) && tap_hits<K, S>(b, kx, c)) {
                  if (DGRAD) {
                    const float4 wv = *reinterpret_cast<const float4*>(s_w + tp * CT + cg * 4);
                    da2[a][b][0] = ffma2(dlo, make_float2(wv.x, wv.y), da2[a][b][0]);
                    da2[a][b][1] = ffma2(dhi, make_float2(wv.z, wv.w), da2[a][b][1]);
                  }
                  if (tp >= TAP0 && tp < TAP1) {
                    gw[tp - TAP0][0] = ffma2(dlo, a1p[a][b][0], gw[tp - TAP0][0]);
                    gw[tp - TAP0][1] = ffma2(dhi, a1p[a][b][1], gw[tp - TAP0][1]);
                  }
                }
              }
            }
          }
        }
      }
    }
    if (DGRAD) {
      const float4 mu = *reinterpret_cast<const float4*>(s_tab + 5 * CT + cg * 4);
      const float4 rs = *reinterpret_cast<const float4*>(s_tab + 6 * CT + cg * 4);
      const float4 nmr = make_float4(-mu.x * rs.x, -mu.y * rs.y, -mu.z * rs.z, -mu.w * rs.w);
      const size_t img_in = (size_t)n * p.H * p.W * p.ldc + c0;
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          if (!valid[a][b]) continue;
          const uint2 xr = *reinterpret_cast<const uint2*>(xbase + (a * TIW + b) * CT);
          const float xv[4] = {bf16lo(xr.x), bf16hi(xr.x), bf16lo(xr.y), bf16hi(xr.y)};
          const float z[4] = {fmaf(sc.x, xv[0], sh.x), fmaf(sc.y, xv[1], sh.y),
                              fmaf(sc.z, xv[2], sh.z), fmaf(sc.w, xv[3], sh.w)};
          float da[4] = {da2[a][b][0].x, da2[a][b][0].y, da2[a][b][1].x, da2[a][b][1].y};
          act_bwd_vec<4>(da, z, ap, act);
          const size_t off = img_in + (unsigned)(((y0 + py + a) * p.W + x0 + px + b) * p.ldc);
          if (p.residual) {
            float rv[4];
            ld4(p.residual + off, rv);
#pragma unroll
            for (int v = 0; v < 4; ++v) da[v] += rv[v];
          }
          *reinterpret_cast<uint2*>(p.dx + off) =
              make_uint2(pack_bf16(da[0], da[1]), pack_bf16(da[2], da[3]));
          // statistics of the fp32 values (see the forward kernel); xhat = x*rs - mu*rs
          ssum[0] += da[0]; ssum[1] += da[1]; ssum[2] += da[2]; ssum[3] += da[3];
          ssq[0] = fmaf(da[0], fmaf(xv[0], rs.x, nmr.x), ssq[0]);
          ssq[1] = fmaf(da[1], fmaf(xv[1], rs.y, nmr.y), ssq[1]);
          ssq[2] = fmaf(da[2], fmaf(xv[2], rs.z, nmr.z), ssq[2]);
          ssq[3] = fmaf(da[3], fmaf(xv[3], rs.w, nmr.w), ssq[3]);
        }
    }
  }
  cp_async_wait<0>();
  if (cur_chunk >= 0) flush(cur_chunk);
  if (p.has_bn && DGRAD) {
    if (arrive_last(p.bn.counter)) {
      bn_bwd_finalize(p.bn, p.C);
      __syncthreads();
      if (threadIdx.x == 0) *p.bn.counter = 0;
    }
  }
}

// Grid of kernel `kern` for `tiles` tiles at `smem` bytes of dynamic shared memory.
template <typename Kern, typename Dev>
static cudaError_t grid_k(Kern kern, const Dev& p, size_t smem, long long tiles, int* grid_out) {
  // The dynamic-smem limit of a kernel is process-wide state: only ever RAISE it (forward and
  // backward run on different host threads); occupancy is cached per (kernel, smem size).
  struct Ent { const void* k; size_t smem; int per_sm; };
  static Ent cache[128];
  static int n_cache = 0;
  static std::mutex mu;
  int per_sm = 0;
  {
    std::lock_guard<std::mutex> lock(mu);
    size_t limit = 0;
    for (int i = 0; i < n_cache; ++i)
      if (cache[i].k == (const void*)kern) {
        if (cache[i].smem > limit) limit = cache[i].smem;
        if (cache[i].smem == smem) per_sm = cache[i].per_sm;
      }
    if (per_sm == 0) {
      cudaError_t e;
      if (smem > limit) {
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
      }
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, smem);
      if (e != cudaSuccess) return e;
      if (per_sm < 1) return cudaErrorLaunchOutOfResources;
      if (n_cache < 128) cache[n_cache++] = Ent{(const void*)kern, smem, per_sm};
    }
  }
  long long cap = (long long)max_ctas() * (per_sm > 4 ? 4 : per_sm);  // partials sized for 4/SM
  int grid = (int)(tiles < cap ? tiles : cap);
  // Tiles are ordered channel-chunk-major and every CTA walks a contiguous range.  With a grid that
  // is a multiple of the chunk count, CTA b and CTA b + grid/chunks walk the SAME spatial tiles of
  // neighbouring channel chunks at the same time, so the 128-byte lines that straddle two chunks
  // (pixels of 192 / 288 bytes read in 64-byte pieces) and the halo rows are served by L2 instead
  // of being fetched from DRAM once per chunk (ncu r01: 2.7x the algorithmic reads at C = 144).
  if (p.chunks > 1 && grid > p.chunks) grid = grid / p.chunks * p.chunks;
  if (grid < 1) grid = 1;
  *grid_out = grid;
  return cudaSuccess;
}

template <typename Kern, typename Dev>
static cudaError_t launch_k(Kern kern, const Dev& p, size_t smem, long long tiles, cudaStream_t st) {
  int grid = 0;
  cudaError_t e = grid_k(kern, p, smem, tiles, &grid);
  if (e != cudaSuccess) return e;
  kern<<<grid, 256, smem, st>>>(p);
  return cudaGetLastError();
}

template <int KK, int SS, int CC, typename Dev>
static cudaError_t launch_bwd(const Dev& p0, size_t smem, long long tiles, cudaStream_t st) {
  // weight gradient: per-CTA partials (zero where a CTA has no tile of a channel chunk), then
  // added in CTA order
  auto k0 = dw_bwd_kernel<KK, SS, CC, 0, (KK == 7 ? 25 : KK * KK), true>;
  int g0 = 0, g1 = 0;
  cudaError_t e = grid_k(k0, p0, smem, tiles, &g0);
  if constexpr (KK == 7)   // the taps past 25 in a second kernel
    if (e == cudaSuccess) e = grid_k(dw_bwd_kernel<KK, SS, CC, 25, KK * KK, false>, p0, smem, tiles, &g1);
  if (e != cudaSuccess) return e;
  const int slabs = g0 > g1 ? g0 : g1;
  const long long n = (long long)p0.C * KK * KK;
  Dev p = p0;
  if (det_alloc((size_t)(slabs * n) * sizeof(float), st, &p.part)) return cudaErrorMemoryAllocation;
  e = cudaMemsetAsync(p.part, 0, (size_t)(slabs * n) * sizeof(float), st);
  if (e == cudaSuccess) {
    k0<<<g0, 256, smem, st>>>(p);
    e = cudaGetLastError();
  }
  if constexpr (KK == 7) {
    if (e == cudaSuccess) {
      dw_bwd_kernel<KK, SS, CC, 25, KK * KK, false><<<g1, 256, smem, st>>>(p);
      e = cudaGetLastError();
    }
  }
  if (e != cudaSuccess) {
    det_free(p.part, st);
    return e;
  }
  if (det_reduce_launch(p.part, slabs, n, p.dw, st)) return cudaErrorLaunchFailure;
  return cudaSuccess;
}
#define YAMB_DW_BWD(KK, SS, CC, ...) e = launch_bwd<KK, SS, CC>(__VA_ARGS__)


// 8 / 16-channel tiles (depthwise_narrow.cu); cudaErrorInvalidValue when the combination is not built
cudaError_t dw_fwd_dispatch_narrow(const DwFwdDev& p, int k, int s, int ct, int tw, size_t smem,
                                   cudaStream_t st);
cudaError_t dw_bwd_dispatch_narrow(const DwBwdDev& p, int k, int s, int ct, size_t smem,
                                   cudaStream_t st);

}  // namespace yamb
