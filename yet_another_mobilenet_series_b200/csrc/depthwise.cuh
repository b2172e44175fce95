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
#include <cuda_runtime.h>

#include "bn_finalize.cuh"
#include "host_util.h"
#include "prims.cuh"

namespace yamb {

// resident CTAs per SM the 3x3 kernels are compiled for (register cap 64 Ki / (256 * n))
constexpr int kDw3MinBlocks = 2;

__device__ __forceinline__ void ld4(const __nv_bfloat16* p, float (&v)[4]) {
  const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
  v[0] = bf16lo(u.x); v[1] = bf16hi(u.x); v[2] = bf16lo(u.y); v[3] = bf16hi(u.y);
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

// Forward, v4: the raw bf16 input tile (with halo) of tile t+1 streams into shared memory with
// cp.async (zero-fill outside the image) while tile t is transformed IN PLACE (BN + activation,
// rounded to bf16 like every other materialised activation) and convolved.
template <int K, int S, int CT, int TW>
__global__ void __launch_bounds__(256, (K == 3 ? kDw3MinBlocks : 1)) dw_fwd_kernel(
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
        cp_async_zfill16(dst + k * PSTEP * CT * 2, src, ok ? 16 : 0);
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

// Squeeze-and-Excitation operands of the depthwise backward of an SE block (pre-offset to the slice)
struct DwSeDev {
  const float* gate;    // [N][ldg]
  const float* dpool;   // [N][ldg]
  int ldg;
  const float *scale, *shift;   // BatchNorm-2 coefficients: z2 = scale*h + shift
  int act;
};

struct DwBwdSeDev {
  DwBwdDev dw;
  DwSeDev se;
};

// dz = bf16((dY * gate[n][c] + dpool[n][c]) * act'(scale * h + shift)) of the 8 channels c8.. of a
// staged vector: the fp32 operations and rounding of se_bwd_apply_kernel
__device__ __forceinline__ uint4 se_dz(const uint4& rdy, const uint4& rh, const DwSeDev& se, int n,
                                       int c8) {
  float d[8], hv[8], g[8], pp[8], sc[8], sh[8];
  unpack8(rdy, d);
  unpack8(rh, hv);
  const float4* g4 = reinterpret_cast<const float4*>(se.gate + (size_t)n * se.ldg + c8);
  const float4* d4 = reinterpret_cast<const float4*>(se.dpool + (size_t)n * se.ldg + c8);
  const float4* s4 = reinterpret_cast<const float4*>(se.scale + c8);
  const float4* t4 = reinterpret_cast<const float4*>(se.shift + c8);
#pragma unroll
  for (int v = 0; v < 2; ++v) {
    const float4 a = __ldg(g4 + v), b = __ldg(d4 + v), c = __ldg(s4 + v), e = __ldg(t4 + v);
    g[4 * v] = a.x; g[4 * v + 1] = a.y; g[4 * v + 2] = a.z; g[4 * v + 3] = a.w;
    pp[4 * v] = b.x; pp[4 * v + 1] = b.y; pp[4 * v + 2] = b.z; pp[4 * v + 3] = b.w;
    sc[4 * v] = c.x; sc[4 * v + 1] = c.y; sc[4 * v + 2] = c.z; sc[4 * v + 3] = c.w;
    sh[4 * v] = e.x; sh[4 * v + 1] = e.y; sh[4 * v + 2] = e.z; sh[4 * v + 3] = e.w;
  }
  const ActParam ap = make_act(se.act);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float z = fmaf(sc[e], hv[e], sh[e]);
    d[e] = fmaf(d[e], g[e], pp[e]) * act_bwd_rt(z, ap, se.act);
  }
  return pack8(d);
}

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
#define YAMB_DW_BWD_SE 0
#include "depthwise_bwd_kernel.cuh"
#undef YAMB_DW_BWD_SE
#define YAMB_DW_BWD_SE 1
#include "depthwise_bwd_kernel.cuh"
#undef YAMB_DW_BWD_SE

// Grid of kernel `kern` for `tiles` tiles at `smem` bytes of dynamic shared memory.
template <typename Kern, typename Dev>
static int grid_k(const char* fn, Kern kern, const Dev& p, size_t smem, long long tiles,
                  int* grid_out) {
  int per_sm = 0;
  int rc = smem_optin(fn, (const void*)kern, smem, &per_sm);
  if (rc) return rc;
  if (per_sm < 1) return set_error(YAMB_ECUDA, "%s: no CTA fits on an SM", fn);
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
  return 0;
}

// The launchers below return 0 or a YAMB_* code with the message set.
template <typename Kern, typename Dev>
static int launch_k(Kern kern, const Dev& p, size_t smem, long long tiles, cudaStream_t st) {
  int grid = 0;
  int rc = grid_k("dw fwd launch", kern, p, smem, tiles, &grid);
  if (rc) return rc;
  kern<<<grid, 256, smem, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "dw fwd launch: %s", cudaGetErrorString(e));
  return 0;
}

// the backward kernel of an argument type: DwBwdDev (dw_bwd_kernel) or DwBwdSeDev (dw_bwd_se_kernel)
template <int K, int S, int CT, int TAP0, int TAP1, bool DGRAD>
struct BwdKernel {
  static constexpr auto of(const DwBwdDev*) { return dw_bwd_kernel<K, S, CT, TAP0, TAP1, DGRAD>; }
  static constexpr auto of(const DwBwdSeDev*) { return dw_bwd_se_kernel<K, S, CT, TAP0, TAP1, DGRAD>; }
};
static inline DwBwdDev& dw_core(DwBwdDev& p) { return p; }
static inline DwBwdDev& dw_core(DwBwdSeDev& p) { return p.dw; }

template <int KK, int SS, int CC, typename Dev>
static int launch_bwd(const Dev& p0, size_t smem, long long tiles, cudaStream_t st) {
  // weight gradient: per-CTA partials (zero where a CTA has no tile of a channel chunk), then
  // added in CTA order
  auto k0 = BwdKernel<KK, SS, CC, 0, (KK == 7 ? 25 : KK * KK), true>::of(&p0);
  Dev p = p0;
  DwBwdDev& core = dw_core(p);
  int g0 = 0, g1 = 0;
  int rc = grid_k("dw bwd launch", k0, core, smem, tiles, &g0);
  if constexpr (KK == 7)   // the taps past 25 in a second kernel
    if (!rc) rc = grid_k("dw bwd launch", BwdKernel<KK, SS, CC, 25, KK * KK, false>::of(&p0), core,
                         smem, tiles, &g1);
  if (rc) return rc;
  const int slabs = g0 > g1 ? g0 : g1;
  const long long n = (long long)core.C * KK * KK;
  if ((rc = det_alloc((size_t)(slabs * n) * sizeof(float), st, &core.part))) return rc;
  cudaError_t e = cudaMemsetAsync(core.part, 0, (size_t)(slabs * n) * sizeof(float), st);
  if (e == cudaSuccess) {
    k0<<<g0, 256, smem, st>>>(p);
    e = cudaGetLastError();
  }
  if constexpr (KK == 7) {
    if (e == cudaSuccess) {
      BwdKernel<KK, SS, CC, 25, KK * KK, false>::of(&p0)<<<g1, 256, smem, st>>>(p);
      e = cudaGetLastError();
    }
  }
  if (e != cudaSuccess) {
    det_free(core.part, st);
    return set_error(YAMB_ECUDA, "dw bwd launch: %s", cudaGetErrorString(e));
  }
  return det_reduce_launch(core.part, slabs, n, core.dw, st);
}
#define YAMB_DW_BWD(KK, SS, CC, ...) rc = launch_bwd<KK, SS, CC>(__VA_ARGS__)


// 8 / 16-channel tiles (depthwise_narrow.cu); YAMB_ECUDA when the combination is not built
int dw_fwd_dispatch_narrow(const DwFwdDev& p, int k, int s, int ct, int tw, size_t smem,
                           cudaStream_t st);
int dw_bwd_dispatch_narrow(const DwBwdDev& p, int k, int s, int ct, size_t smem, cudaStream_t st);

// Checks the arguments of a depthwise backward and fills the kernel arguments, the channel tile and
// the dynamic shared memory (depthwise.cu): 0, YAMB_EINVAL, or YAMB_ENODEV without a device.
int dw_bwd_setup(const yamb_dw_bwd* a, DwBwdDev* p, int* ct, size_t* smem);

// The dispatch over (k, stride, channel tile) of the SE depthwise backward: 32 / 64-channel tiles in
// depthwise_se.cu, 8 / 16 in depthwise_se_narrow.cu
int dw_bwd_se_dispatch(const DwBwdSeDev& p, int k, int s, int ct, size_t smem, cudaStream_t st);
int dw_bwd_se_dispatch_narrow(const DwBwdSeDev& p, int k, int s, int ct, size_t smem,
                              cudaStream_t st);

}  // namespace yamb
