// Stem convolution: 3x3, stride 2, pad 1, 3 input channels (RGB) -> Cout (<= 64, multiple of 8)
// on NHWC bf16, sm_90a.
//
// Replaces, behind yamb_stem_conv_fwd / yamb_stem_conv_wgrad (include/yamb200.h), the cuDNN
// implicit-GEMM forward / weight-gradient kernels (and the nhwcAddPadding copies cuDNN needs for a
// 3-channel NHWC tensor) that round 1 used for the first layer of the network
// (reference models/mobilenet_supernet.py:124-130: ConvBNReLU(3, input_channel, stride=2)).
// No input gradient: the images do not require one.
//
// forward : thread = 2 horizontally adjacent output pixels x all output channels (8 at a time);
//           the 3x5x3 input patch sits in registers, the weights are broadcast from shared memory.
//           Eval variant (yamb_stem_conv_eval_fwd): the same kernel with the folded BatchNorm +
//           activation applied before the store, so h never reaches HBM.
// wgrad   : dW[co][ci][ky][kx] = sum_pixels dh[p][co] * x[2p+tap][ci]; thread = (pair of output
//           channels, 2 of the 27 (tap, ci) positions); tiles of 16 x 32 output pixels are staged in
//           shared memory; per-thread register accumulators over the CTA's tiles, one fp32
//           reduction per weight element per CTA at the end.
// 864 MACs per output pixel against 6 + 64 bytes of traffic: FMA/LDS bound, not HBM bound.
//
// uint8 input (yamb_stem_conv_u8_*): every kernel also takes x as uint8 HWC bytes and stages
// bf16(((float)u / 255 - mean[c]) / std[c]) (torchvision's ToTensor + Normalize, then the bf16
// rounding of the bf16 path) into the same shared-memory tile, 0 outside the image; the normalised
// values come from a [3][256] table each CTA builds once.  From the staged tile on, the code is
// that of the bf16 instantiation, so the results are bitwise those of the bf16 entry points on the
// host-normalised image.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cmath>
#include <type_traits>

#include "host_util.h"
#include "prims.cuh"

namespace yamb {

constexpr int kStemTH = 16, kStemTW = 32;            // output tile
constexpr int kStemIH = 2 * kStemTH + 1, kStemIW = 2 * kStemTW + 1;   // input tile incl. halo

template <typename T>
constexpr bool kStemU8 = std::is_same<T, uint8_t>::value;
constexpr size_t kStemLutBytes = 3 * 256 * 2;          // uint8 input: [c][u] normalised bf16

struct StemDev {
  int N, H, W, Ho, Wo, Cout;
  const void* x;              // [N][H][W][3] bf16, or uint8 for the uint8 instantiations
  const float* w;             // [Cout][3][3][3]
  __nv_bfloat16* y;           // [N][Ho][Wo][Cout]        (forward)
  const __nv_bfloat16* dh;    // [N][Ho][Wo][Cout]        (wgrad)
  float* dw;                  // [Cout][3][3][3] +=       (wgrad)
  float* part;                // [CTA x pixel subset][Cout][27] wgrad partials
  int tiles_h, tiles_w, num_tiles;
  const float* scale;         // [Cout] eval forward: y = act(scale * bf16(conv) + shift)
  const float* shift;
  int act;
  float mean[3], stdv[3];     // uint8 input: x_staged = bf16(((float)u / 255 - mean[c]) / stdv[c])
};

// The staged input tile starts ONE pixel left of the halo (column ix0 - 1) so that, with the tile
// origin at an even pixel, every row segment begins on a 4-byte boundary and is copied as 32-bit
// words: s_in[IH][kStemSW][3], input pixel ix lives at column ix - (ix0 - 1).
constexpr int kStemSW = kStemIW + 1;                  // 66 staged columns
constexpr int kStemRowWords = kStemSW * 3 / 2;        // 99 words per staged row

// All copies of a tile are issued as asynchronous 4-byte cp.async (zero-filled outside the image)
// and awaited ONCE by the caller (commit, then wait): a plain load loop exposed one DRAM round
// trip per iteration, 13 per tile.
__device__ __forceinline__ void stem_stage_input(const StemDev& p, int n, int ty, int tx,
                                                 __nv_bfloat16* s_in) {
  const int iy0 = ty * kStemTH * 2 - 1, ixs = tx * kStemTW * 2 - 2;   // ixs even
  const __nv_bfloat16* img = static_cast<const __nv_bfloat16*>(p.x) + (size_t)n * p.H * p.W * 3;
  uint32_t* dst = reinterpret_cast<uint32_t*>(s_in);
#pragma unroll 1
  for (int e = threadIdx.x; e < kStemIH * kStemRowWords; e += 256) {
    const int r = e / kStemRowWords, wd = e - r * kStemRowWords;
    const int iy = iy0 + r;
    // elements 2*wd, 2*wd+1 of the row's (pixel, channel) sequence starting at pixel ixs
    const int k0 = 2 * wd;
    const int px0 = ixs + k0 / 3, px1 = ixs + (k0 + 1) / 3;
    const bool rowok = (unsigned)iy < (unsigned)p.H;
    const bool v0 = rowok && px0 >= 0 && px0 < p.W, v1 = rowok && px1 >= 0 && px1 < p.W;
    const __nv_bfloat16* src = img + (size_t)(rowok ? iy : 0) * p.W * 3 + ((long long)ixs * 3 + k0);
    if (v0 == v1) {        // whole word inside (copy) or outside (zero-fill): 4-byte aligned
      asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst + e)),
                   "l"(v0 ? (const void*)src : (const void*)img), "r"(v0 ? 4 : 0)
                   : "memory");
    } else {               // image border inside the word (odd widths only)
      const uint16_t lo = v0 ? *reinterpret_cast<const uint16_t*>(src) : 0;
      const uint16_t hi = v1 ? *reinterpret_cast<const uint16_t*>(src + 1) : 0;
      dst[e] = (uint32_t)lo | ((uint32_t)hi << 16);
    }
  }
}

// generic 2-byte path (odd image widths)
__device__ __forceinline__ void stem_stage_generic(const StemDev& p, int n, int ty, int tx,
                                                   __nv_bfloat16* s_in) {
  const int iy0 = ty * kStemTH * 2 - 1, ixs = tx * kStemTW * 2 - 2;
  const __nv_bfloat16* img = static_cast<const __nv_bfloat16*>(p.x) + (size_t)n * p.H * p.W * 3;
  for (int e = threadIdx.x; e < kStemIH * kStemSW * 3; e += 256) {
    const int rr = e / (kStemSW * 3), rem = e % (kStemSW * 3);
    const int iy = iy0 + rr, ix = ixs + rem / 3;
    __nv_bfloat16 v = __float2bfloat16(0.f);
    if ((unsigned)iy < (unsigned)p.H && (unsigned)ix < (unsigned)p.W)
      v = img[((size_t)iy * p.W + ix) * 3 + rem % 3];
    s_in[e] = v;
  }
}

// ---- uint8 input ----------------------------------------------------------------------------------
// lut[c * 256 + u] = bf16 bits of ((float)u / 255 - mean[c]) / std[c], IEEE-rounded at each step
// as torchvision's fp32 ToTensor + Normalize round on the host.  One entry per thread and channel.
__device__ __forceinline__ void stem_u8_table(const StemDev& p, uint16_t* lut) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = __fdiv_rn(__fsub_rn(__fdiv_rn((float)threadIdx.x, 255.f), p.mean[c]), p.stdv[c]);
    lut[c * 256 + threadIdx.x] = __bfloat16_as_ushort(__float2bfloat16_rn(v));
  }
}

// W % 4 == 0: a row is 3W bytes, so rows and the image's edges fall on 4-byte boundaries.  The
// staged elements k = 0..197 of a tile row (pixel ixs + k / 3, channel k % 3) sit at row bytes
// 3 ixs + k, and 3 ixs = 2 mod 4: 50 aligned words cover them, word 0 starting at element -2.  All
// words of a tile go to a byte buffer by one batch of 4-byte cp.async (zero-filled outside the
// image, awaited once by the caller, as the bf16 path), then stem_u8_convert writes the normalised
// tile.  A word lies wholly inside or wholly outside the image.
constexpr int kStemU8RowWords = 50;
constexpr int kStemU8Words = kStemIH * kStemU8RowWords;
constexpr size_t kStemU8Smem = kStemLutBytes + (size_t)kStemU8Words * 4;   // table + byte tile

__device__ __forceinline__ void stem_u8_issue(const StemDev& p, int n, int ty, int tx,
                                              unsigned char* s_bytes) {
  const int iy0 = ty * kStemTH * 2 - 1;
  const int off0 = (tx * kStemTW * 2 - 2) * 3 - 2;                  // row byte of word 0
  const unsigned char* img = static_cast<const unsigned char*>(p.x) + (size_t)n * p.H * p.W * 3;
#pragma unroll 1
  for (int e = threadIdx.x; e < kStemU8Words; e += 256) {
    const int r = e / kStemU8RowWords, off = off0 + 4 * (e - r * kStemU8RowWords);
    const int iy = iy0 + r;
    const bool ok = (unsigned)iy < (unsigned)p.H && (unsigned)off < (unsigned)(3 * p.W);
    const unsigned char* src = ok ? img + (size_t)iy * p.W * 3 + off : img;
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(s_bytes + 4 * e)),
                 "l"(src), "r"(ok ? 4 : 0)
                 : "memory");
  }
}

// byte tile -> s_in, two elements (one 32-bit word of s_in) per step; the padding is 0, not the
// normalised 0 byte
__device__ __forceinline__ void stem_u8_convert(const StemDev& p, int ty, int tx,
                                                const unsigned char* s_bytes, const uint16_t* lut,
                                                __nv_bfloat16* s_in) {
  const int iy0 = ty * kStemTH * 2 - 1, ixs = tx * kStemTW * 2 - 2;
  uint32_t* dst = reinterpret_cast<uint32_t*>(s_in);
#pragma unroll 1
  for (int q = threadIdx.x; q < kStemIH * kStemRowWords; q += 256) {
    const int r = q / kStemRowWords, k = 2 * (q - r * kStemRowWords);
    const bool rowok = (unsigned)(iy0 + r) < (unsigned)p.H;
    const uint32_t u =
        *reinterpret_cast<const uint16_t*>(s_bytes + r * (4 * kStemU8RowWords) + k + 2);
    const int c0 = k % 3, c1 = c0 == 2 ? 0 : c0 + 1;
    const uint32_t lo =
        rowok && (unsigned)(ixs + k / 3) < (unsigned)p.W ? lut[c0 * 256 + (u & 255)] : 0u;
    const uint32_t hi =
        rowok && (unsigned)(ixs + (k + 1) / 3) < (unsigned)p.W ? lut[c1 * 256 + (u >> 8)] : 0u;
    dst[q] = lo | (hi << 16);
  }
}

// any other width: element by element
__device__ __forceinline__ void stem_u8_stage_generic(const StemDev& p, int n, int ty, int tx,
                                                      const uint16_t* lut, __nv_bfloat16* s_in) {
  const int iy0 = ty * kStemTH * 2 - 1, ixs = tx * kStemTW * 2 - 2;
  const unsigned char* img = static_cast<const unsigned char*>(p.x) + (size_t)n * p.H * p.W * 3;
  uint16_t* dst = reinterpret_cast<uint16_t*>(s_in);
#pragma unroll 1
  for (int e = threadIdx.x; e < kStemIH * kStemSW * 3; e += 256) {
    const int rr = e / (kStemSW * 3), rem = e % (kStemSW * 3);
    const int iy = iy0 + rr, ix = ixs + rem / 3, c = rem % 3;
    uint16_t v = 0;
    if ((unsigned)iy < (unsigned)p.H && (unsigned)ix < (unsigned)p.W)
      v = lut[c * 256 + img[((size_t)iy * p.W + ix) * 3 + c]];
    dst[e] = v;
  }
}

// the aligned staging path of each input type
template <typename T>
__device__ __forceinline__ bool stem_aligned(const StemDev& p) {
  if constexpr (kStemU8<T>)
    return (p.W % 4) == 0 && (reinterpret_cast<uintptr_t>(p.x) & 3) == 0;
  else
    return ((p.W * 3) % 2) == 0;     // odd W*3: rows are only 2-byte aligned
}

// EVAL: the BatchNorm (running statistics folded into scale / shift) and the activation are applied
// between the accumulators and the staging, with the expression and rounding points of
// bn_apply_kernel (elementwise.cu): y = bf16(act(fmaf(scale, bf16(conv), shift))).
// T: the type of x (__nv_bfloat16, or uint8_t normalised while it is staged).
template <bool EVAL, typename T>
__device__ __forceinline__ void stem_fwd_body(const StemDev& p) {
  extern __shared__ __align__(16) unsigned char stem_smem[];
  float* s_w = reinterpret_cast<float*>(stem_smem);                // [tap*3+ci][co], 27*64 floats
  __nv_bfloat16* s_in = reinterpret_cast<__nv_bfloat16*>(s_w + 27 * 64);   // [IH][SW][3]
  // per-warp output staging: 2 output rows x 32 pixels x Cout channels, written back as whole
  // 16-byte-per-lane coalesced rows (a thread's own 2 x Cout values are 128 B apart from its
  // neighbour's: stored directly, every instruction touched 32 half-used sectors)
  uint4* s_out = reinterpret_cast<uint4*>(s_in + ((kStemIH * kStemSW * 3 + 7) & ~7)) +
                 (threadIdx.x >> 5) * (64 * (p.Cout / 8));
  for (int e = threadIdx.x; e < 27 * p.Cout; e += 256) {
    const int co = e / 27, j = e % 27;           // w[co][ci][ky][kx]: j = ci*9 + ky*3 + kx
    const int ci = j / 9, tap = j % 9;
    s_w[(tap * 3 + ci) * p.Cout + co] = p.w[e];
  }
  // uint8 x: table and byte tile after the 8 warps' output staging
  uint16_t* s_lut = nullptr;
  unsigned char* s_bytes = nullptr;
  if constexpr (kStemU8<T>) {
    s_lut = reinterpret_cast<uint16_t*>(reinterpret_cast<uint4*>(
                s_in + ((kStemIH * kStemSW * 3 + 7) & ~7)) + 8 * 64 * (p.Cout / 8));
    s_bytes = reinterpret_cast<unsigned char*>(s_lut + 3 * 256);
    stem_u8_table(p, s_lut);
  }
  const int ry = threadIdx.x / 16, cp = threadIdx.x % 16;          // output row, column pair
  const bool aligned = stem_aligned<T>(p);
  for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
    const int n = t / (p.tiles_h * p.tiles_w), r = t % (p.tiles_h * p.tiles_w);
    const int ty = r / p.tiles_w, tx = r % p.tiles_w;
    __syncthreads();
    if constexpr (kStemU8<T>) {
      if (aligned) {
        stem_u8_issue(p, n, ty, tx, s_bytes);
        cp_async_commit();
        cp_async_wait<0>();
        __syncthreads();
        stem_u8_convert(p, ty, tx, s_bytes, s_lut, s_in);
      } else {
        stem_u8_stage_generic(p, n, ty, tx, s_lut, s_in);
      }
    } else if (aligned) {
      stem_stage_input(p, n, ty, tx, s_in);
      cp_async_commit();
      cp_async_wait<0>();
    } else {
      stem_stage_generic(p, n, ty, tx, s_in);
    }
    __syncthreads();
    // 3 x 5 x 3 input patch of this thread's two output pixels, as (a, a) pairs for the pair FMAs
    float in[3][5][3];
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 5; ++b)
#pragma unroll
        for (int c = 0; c < 3; ++c)
          in[a][b][c] = __bfloat162float(s_in[((2 * ry + a) * kStemSW + 4 * cp + b + 1) * 3 + c]);
    const int V = p.Cout / 8;                       // 16-byte vectors per pixel
    const int lane = threadIdx.x & 31;
    const int hp = lane >> 4;                       // which of the warp's two output rows
    for (int c0 = 0; c0 < p.Cout; c0 += 8) {
      float2 acc[2][4];
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[0][e] = acc[1][e] = make_float2(0.f, 0.f);
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx)
#pragma unroll
          for (int ci = 0; ci < 3; ++ci) {
            const float4 w0 = *reinterpret_cast<const float4*>(s_w + ((ky * 3 + kx) * 3 + ci) * p.Cout + c0);
            const float4 w1 = *reinterpret_cast<const float4*>(s_w + ((ky * 3 + kx) * 3 + ci) * p.Cout + c0 + 4);
            const float2 wv[4] = {make_float2(w0.x, w0.y), make_float2(w0.z, w0.w),
                                  make_float2(w1.x, w1.y), make_float2(w1.z, w1.w)};
            const float2 a0 = make_float2(in[ky][kx][ci], in[ky][kx][ci]);
            const float2 a1 = make_float2(in[ky][kx + 2][ci], in[ky][kx + 2][ci]);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              acc[0][e] = ffma2(a0, wv[e], acc[0][e]);
              acc[1][e] = ffma2(a1, wv[e], acc[1][e]);
            }
          }
      if (EVAL) {
        const ActParam ap = make_act(p.act);
        float z0[8], z1[8];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          z0[2 * e] = fmaf(p.scale[c0 + 2 * e], round_bf16(acc[0][e].x), p.shift[c0 + 2 * e]);
          z0[2 * e + 1] = fmaf(p.scale[c0 + 2 * e + 1], round_bf16(acc[0][e].y), p.shift[c0 + 2 * e + 1]);
          z1[2 * e] = fmaf(p.scale[c0 + 2 * e], round_bf16(acc[1][e].x), p.shift[c0 + 2 * e]);
          z1[2 * e + 1] = fmaf(p.scale[c0 + 2 * e + 1], round_bf16(acc[1][e].y), p.shift[c0 + 2 * e + 1]);
        }
        act_vec<8>(z0, ap);
        act_vec<8>(z1, ap);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          acc[0][e] = make_float2(z0[2 * e], z0[2 * e + 1]);
          acc[1][e] = make_float2(z1[2 * e], z1[2 * e + 1]);
        }
      }
      // staging layout: [row hp][pixel 0..31][V vectors]
      uint4* so = s_out + (hp * 32 + 2 * cp) * V + (c0 >> 3);
      so[0] = make_uint4(pack_bf16(acc[0][0].x, acc[0][0].y), pack_bf16(acc[0][1].x, acc[0][1].y),
                         pack_bf16(acc[0][2].x, acc[0][2].y), pack_bf16(acc[0][3].x, acc[0][3].y));
      so[V] = make_uint4(pack_bf16(acc[1][0].x, acc[1][0].y), pack_bf16(acc[1][1].x, acc[1][1].y),
                         pack_bf16(acc[1][2].x, acc[1][2].y), pack_bf16(acc[1][3].x, acc[1][3].y));
    }
    __syncwarp();
    // the warp's two rows: oy = tile row (2 * warp + hp'), 32 pixels x V vectors each, contiguous
    const int wrow = (threadIdx.x >> 5) * 2;
    const int ox0 = tx * kStemTW;
    for (int q = lane; q < 64 * V; q += 32) {
      const int rr = q / (32 * V), within = q - rr * 32 * V;     // row, vector inside the row
      const int oy = ty * kStemTH + wrow + rr, ox = ox0 + within / V;
      if (oy < p.Ho && ox < p.Wo)
        reinterpret_cast<uint4*>(p.y + (((size_t)n * p.Ho + oy) * p.Wo + ox0) * p.Cout)[within] =
            s_out[q];
    }
    __syncwarp();
  }
}

template <bool EVAL>
__global__ void __launch_bounds__(256) stem_fwd_kernel(const __grid_constant__ StemDev p) {
  stem_fwd_body<EVAL, __nv_bfloat16>(p);
}
// uint8 x: at the default bound the training forward took 104 registers (the bf16 one 80), two
// CTAs per SM instead of three; min-blocks 3 holds it at 80 without spills.  The eval forward
// keeps the 128 registers of its bf16 twin.
template <bool EVAL>
__global__ void __launch_bounds__(256, EVAL ? 2 : 3) stem_fwd_u8_kernel(
    const __grid_constant__ StemDev p) {
  stem_fwd_body<EVAL, uint8_t>(p);
}

// wgrad: thread = (8 output channels co8, 4 positions jq, pixel subset ps): 256 threads =
// (Cout/8) x 8 x PS.  32 FMAs per 2 + 4 shared-memory loads.  Positions are walked in
// staging order jj = (ky*3 + kx)*3 + ci and mapped to the parameter's j = ci*9 + ky*3 + kx at the end.
template <typename T>
__global__ void __launch_bounds__(256) stem_wgrad_kernel(const __grid_constant__ StemDev p) {
  extern __shared__ __align__(16) unsigned char stem_smem[];
  __nv_bfloat16* s_in = reinterpret_cast<__nv_bfloat16*>(stem_smem);          // [IH][SW][3]
  __nv_bfloat16* s_dh = s_in + ((kStemIH * kStemSW * 3 + 7) & ~7);            // [TH*TW][Cout]
  // uint8 x: table and byte tile after s_dh
  uint16_t* s_lut = nullptr;
  unsigned char* s_bytes = nullptr;
  if constexpr (kStemU8<T>) {
    s_lut = reinterpret_cast<uint16_t*>(s_dh + kStemTH * kStemTW * p.Cout);
    s_bytes = reinterpret_cast<unsigned char*>(s_lut + 3 * 256);
    stem_u8_table(p, s_lut);
  }
  const int CO = p.Cout / 8;                        // channel octets (4 for Cout = 32)
  const int PS = 256 / (CO * 8);                    // pixel subsets (8 for Cout = 32)
  const int co8 = threadIdx.x % CO, jq = (threadIdx.x / CO) % 8, ps = threadIdx.x / (CO * 8);
  float2 acc[4][4];
  int joff[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[k][e] = make_float2(0.f, 0.f);
    const int jj = min(4 * jq + k, 26);             // positions 27..31 of the last group: dummies
    const int tap = jj / 3, ci = jj % 3;
    joff[k] = ((tap / 3) * kStemSW + (tap % 3) + 1) * 3 + ci;
  }
  const bool aligned = stem_aligned<T>(p);
  for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
    const int n = t / (p.tiles_h * p.tiles_w), r = t % (p.tiles_h * p.tiles_w);
    const int ty = r / p.tiles_w, tx = r % p.tiles_w;
    __syncthreads();
    if constexpr (kStemU8<T>) {
      if (aligned) stem_u8_issue(p, n, ty, tx, s_bytes);     // converted once the copies land
      else stem_u8_stage_generic(p, n, ty, tx, s_lut, s_in);
    } else if (aligned) {
      stem_stage_input(p, n, ty, tx, s_in);
    } else {
      stem_stage_generic(p, n, ty, tx, s_in);
    }
    // dh tile, zero outside the image: 16-byte vectors
    const int V = p.Cout / 8;
    for (int e = threadIdx.x; e < kStemTH * kStemTW * V; e += 256) {
      const int pix = e / V, v = e % V;
      const int oy = ty * kStemTH + pix / kStemTW, ox = tx * kStemTW + pix % kStemTW;
      const bool ok = oy < p.Ho && ox < p.Wo;
      const void* src = ok ? (const void*)(reinterpret_cast<const uint4*>(
                                 p.dh + (((size_t)n * p.Ho + oy) * p.Wo + ox) * p.Cout) + v)
                           : (const void*)p.dh;
      cp_async_zfill16(smem_u32(reinterpret_cast<uint4*>(s_dh) + e), src, ok ? 16 : 0);
    }
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    if constexpr (kStemU8<T>) {
      if (aligned) {
        stem_u8_convert(p, ty, tx, s_bytes, s_lut, s_in);
        __syncthreads();
      }
    }
#pragma unroll 2
    for (int pix = ps; pix < kStemTH * kStemTW; pix += PS) {
      const uint4 d = reinterpret_cast<const uint4*>(s_dh + (size_t)pix * p.Cout)[co8];
      const float2 dd[4] = {make_float2(bf16lo(d.x), bf16hi(d.x)), make_float2(bf16lo(d.y), bf16hi(d.y)),
                            make_float2(bf16lo(d.z), bf16hi(d.z)), make_float2(bf16lo(d.w), bf16hi(d.w))};
      const int base = ((2 * (pix / kStemTW)) * kStemSW + 2 * (pix % kStemTW)) * 3;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float xv = __bfloat162float(s_in[base + joff[k]]);
        const float2 xx = make_float2(xv, xv);
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[k][e] = ffma2(xx, dd[e], acc[k][e]);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int jj = 4 * jq + k;
    if (jj < 27) {
      const int tap = jj / 3, ci = jj % 3;
      const int j = ci * 9 + tap;
      // partial of (CTA, pixel subset): every slot gets all Cout x 27 values; added in slot order
      float* d = p.part + ((size_t)blockIdx.x * PS + ps) * (p.Cout * 27) + (size_t)(8 * co8) * 27 + j;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        d[(2 * e) * 27] = acc[k][e].x;
        d[(2 * e + 1) * 27] = acc[k][e].y;
      }
    }
  }
}

// Shape checks and the tile plan; touches no device.  Every launcher finishes its own argument
// checks before it looks for a device, so a malformed call is YAMB_EINVAL with or without one.
// u8: the uint8 entry's arguments (their normalisation is checked and copied), or nullptr for bf16.
static int stem_fill(const yamb_stem_conv* a, const yamb_stem_conv_u8* u8, StemDev& p) {
  if (!a || a->N <= 0 || a->H <= 0 || a->W <= 0 || !a->x)
    return set_error(YAMB_EINVAL, "stem conv: bad arguments");
  if (a->Cout <= 0 || a->Cout > 64 || (a->Cout % 8))
    return set_error(YAMB_EINVAL, "stem conv: Cout=%d must be a multiple of 8, <= 64", a->Cout);
  if (u8) {
    for (int c = 0; c < 3; ++c) {
      if (!std::isfinite(u8->mean[c]) || !std::isfinite(u8->std[c]) || u8->std[c] == 0.f)
        return set_error(YAMB_EINVAL, "stem conv u8: mean[%d]=%g, std[%d]=%g: finite, std != 0", c,
                         (double)u8->mean[c], c, (double)u8->std[c]);
      p.mean[c] = u8->mean[c];
      p.stdv[c] = u8->std[c];
    }
  }
  p.N = a->N; p.H = a->H; p.W = a->W; p.Cout = a->Cout;
  p.Ho = (a->H - 1) / 2 + 1; p.Wo = (a->W - 1) / 2 + 1;
  p.x = a->x; p.w = a->w; p.y = (__nv_bfloat16*)a->y;
  p.dh = (const __nv_bfloat16*)a->dh; p.dw = a->dw;
  p.tiles_h = (p.Ho + kStemTH - 1) / kStemTH;
  p.tiles_w = (p.Wo + kStemTW - 1) / kStemTW;
  long long nt = (long long)a->N * p.tiles_h * p.tiles_w;
  if (nt > 0x7fffffffLL) return set_error(YAMB_EINVAL, "stem conv: too many tiles");
  p.num_tiles = (int)nt;
  return 0;
}

template <bool EVAL, typename T>
static int stem_fwd_run(const StemDev& p, int Cout, cudaStream_t st) {
  const size_t smem = 27 * 64 * 4 + (size_t)((kStemIH * kStemSW * 3 + 7) & ~7) * 2 +
                      (size_t)8 * 64 * (Cout / 8) * 16 + (kStemU8<T> ? kStemU8Smem : 0);
  const void* kern = kStemU8<T> ? (const void*)stem_fwd_u8_kernel<EVAL>
                                 : (const void*)stem_fwd_kernel<EVAL>;
  int per_sm = 0;
  const int rc = smem_optin("stem conv fwd", kern, smem, &per_sm);
  if (rc) return rc;
  const int res_f = max_ctas() * (per_sm > 0 ? per_sm : 1);   // one resident wave: no tail
  const int grid = p.num_tiles < res_f ? p.num_tiles : res_f;
  if constexpr (kStemU8<T>) stem_fwd_u8_kernel<EVAL><<<grid, 256, smem, st>>>(p);
  else stem_fwd_kernel<EVAL><<<grid, 256, smem, st>>>(p);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "stem conv fwd: %s", cudaGetErrorString(e));
  return 0;
}

static int stem_fwd(const yamb_stem_conv* a, const yamb_stem_conv_u8* u8, cudaStream_t st) {
  StemDev p;
  int rc = stem_fill(a, u8, p);
  if (rc) return rc;
  if (!a->w || !a->y || (reinterpret_cast<uintptr_t>(a->y) & 15))
    return set_error(YAMB_EINVAL, "stem conv fwd: w / y (16-byte aligned) required");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  p.scale = p.shift = nullptr;
  p.act = 0;
  return u8 ? stem_fwd_run<false, uint8_t>(p, a->Cout, st)
            : stem_fwd_run<false, __nv_bfloat16>(p, a->Cout, st);
}

static int stem_eval_fwd(const yamb_stem_conv_eval* a, const yamb_stem_conv_u8* u8,
                         cudaStream_t st) {
  if (!a) return set_error(YAMB_EINVAL, "stem conv eval: bad arguments");
  StemDev p;
  int rc = stem_fill(&a->conv, u8, p);
  if (rc) return rc;
  if (!a->conv.w || !a->conv.y || (reinterpret_cast<uintptr_t>(a->conv.y) & 15) || !a->scale ||
      !a->shift)
    return set_error(YAMB_EINVAL, "stem conv eval: w / y (16-byte aligned) / scale / shift required");
  if (a->act < YAMB_ACT_NONE || a->act > YAMB_ACT_HSWISH)
    return set_error(YAMB_EINVAL, "stem conv eval: act=%d", a->act);
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  p.scale = a->scale;
  p.shift = a->shift;
  p.act = a->act;
  return u8 ? stem_fwd_run<true, uint8_t>(p, a->conv.Cout, st)
            : stem_fwd_run<true, __nv_bfloat16>(p, a->conv.Cout, st);
}

static int stem_wgrad(const yamb_stem_conv* a, const yamb_stem_conv_u8* u8, cudaStream_t st) {
  StemDev p;
  int rc = stem_fill(a, u8, p);
  if (rc) return rc;
  if (!a->dh || !a->dw || (reinterpret_cast<uintptr_t>(a->dh) & 15))
    return set_error(YAMB_EINVAL, "stem conv wgrad: dh (16-byte aligned) / dw required");
  if (256 % a->Cout) return set_error(YAMB_EINVAL, "stem conv wgrad: Cout must be 8, 16, 32 or 64");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  const size_t smem = (size_t)((kStemIH * kStemSW * 3 + 7) & ~7) * 2 +
                      (size_t)kStemTH * kStemTW * a->Cout * 2;
  // the grid sets the number of partial slabs and so the order of their sum: it comes from the
  // occupancy of the bf16 kernel at this Cout's shared memory, also for a uint8 x, whose kernel
  // (table and byte tile) may hold fewer CTAs per SM: its dw is then bitwise the bf16 kernel's
  int per_sm = 0;
  if ((rc = smem_optin("stem conv wgrad", (const void*)stem_wgrad_kernel<__nv_bfloat16>, smem,
                       &per_sm)))
    return rc;
  if (u8 && (rc = smem_optin("stem conv wgrad", (const void*)stem_wgrad_kernel<uint8_t>,
                             smem + kStemU8Smem)))
    return rc;
  const int res_w = max_ctas() * (per_sm > 0 ? per_sm : 1);
  const int grid = p.num_tiles < res_w ? p.num_tiles : res_w;
  const int slots = grid * (256 / p.Cout);
  rc = det_alloc((size_t)slots * p.Cout * 27 * sizeof(float), st, &p.part);
  if (rc) return rc;
  if (u8) stem_wgrad_kernel<uint8_t><<<grid, 256, smem + kStemU8Smem, st>>>(p);
  else stem_wgrad_kernel<__nv_bfloat16><<<grid, 256, smem, st>>>(p);
  if (cudaPeekAtLastError() != cudaSuccess) det_free(p.part, st);
  else if ((rc = det_reduce_launch(p.part, slots, (long long)p.Cout * 27, p.dw, st)) != 0) return rc;
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "stem conv wgrad: %s", cudaGetErrorString(e));
  return 0;
}

int stem_conv_fwd_launch(const yamb_stem_conv* a, cudaStream_t st) { return stem_fwd(a, nullptr, st); }
int stem_conv_eval_fwd_launch(const yamb_stem_conv_eval* a, cudaStream_t st) {
  return stem_eval_fwd(a, nullptr, st);
}
int stem_conv_wgrad_launch(const yamb_stem_conv* a, cudaStream_t st) { return stem_wgrad(a, nullptr, st); }

int stem_conv_u8_fwd_launch(const yamb_stem_conv_u8* a, cudaStream_t st) {
  if (!a) return set_error(YAMB_EINVAL, "stem conv u8: bad arguments");
  return stem_fwd(&a->ev.conv, a, st);
}
int stem_conv_u8_eval_fwd_launch(const yamb_stem_conv_u8* a, cudaStream_t st) {
  if (!a) return set_error(YAMB_EINVAL, "stem conv u8: bad arguments");
  return stem_eval_fwd(&a->ev, a, st);
}
int stem_conv_u8_wgrad_launch(const yamb_stem_conv_u8* a, cudaStream_t st) {
  if (!a) return set_error(YAMB_EINVAL, "stem conv u8: bad arguments");
  return stem_wgrad(&a->ev.conv, a, st);
}

}  // namespace yamb
