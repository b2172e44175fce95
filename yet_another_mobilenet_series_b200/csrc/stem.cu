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
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "host_util.h"
#include "prims.cuh"

namespace yamb {

constexpr int kStemTH = 16, kStemTW = 32;            // output tile
constexpr int kStemIH = 2 * kStemTH + 1, kStemIW = 2 * kStemTW + 1;   // input tile incl. halo

struct StemDev {
  int N, H, W, Ho, Wo, Cout;
  const __nv_bfloat16* x;     // [N][H][W][3]
  const float* w;             // [Cout][3][3][3]
  __nv_bfloat16* y;           // [N][Ho][Wo][Cout]        (forward)
  const __nv_bfloat16* dh;    // [N][Ho][Wo][Cout]        (wgrad)
  float* dw;                  // [Cout][3][3][3] +=       (wgrad)
  float* part;                // [CTA x pixel subset][Cout][27] wgrad partials
  int tiles_h, tiles_w, num_tiles;
  const float* scale;         // [Cout] eval forward: y = act(scale * bf16(conv) + shift)
  const float* shift;
  int act;
};

// The staged input tile starts ONE pixel left of the halo (column ix0 - 1) so that, with the tile
// origin at an even pixel, every row segment begins on a 4-byte boundary and is copied as 32-bit
// words: s_in[IH][kStemSW][3], input pixel ix lives at column ix - (ix0 - 1).
constexpr int kStemSW = kStemIW + 1;                  // 66 staged columns
constexpr int kStemRowWords = kStemSW * 3 / 2;        // 99 words per staged row

// All copies of a tile are issued as asynchronous 4-byte cp.async (zero-filled outside the image)
// and awaited ONCE by the caller (stem_stage_wait): a plain load loop exposed one DRAM round
// trip per iteration, 13 per tile.
__device__ __forceinline__ void stem_stage_input(const StemDev& p, int n, int ty, int tx,
                                                 __nv_bfloat16* s_in) {
  const int iy0 = ty * kStemTH * 2 - 1, ixs = tx * kStemTW * 2 - 2;   // ixs even
  const __nv_bfloat16* img = p.x + (size_t)n * p.H * p.W * 3;
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
__device__ __forceinline__ void stem_stage_wait() {
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// EVAL: the BatchNorm (running statistics folded into scale / shift) and the activation are applied
// between the accumulators and the staging, with the expression and rounding points of
// bn_apply_kernel (elementwise.cu): y = bf16(act(fmaf(scale, bf16(conv), shift))).
template <bool EVAL>
__global__ void __launch_bounds__(256) stem_fwd_kernel(const __grid_constant__ StemDev p) {
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
  const int ry = threadIdx.x / 16, cp = threadIdx.x % 16;          // output row, column pair
  const bool aligned = ((p.W * 3) % 2) == 0;     // odd W*3: rows are only 2-byte aligned
  for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
    const int n = t / (p.tiles_h * p.tiles_w), r = t % (p.tiles_h * p.tiles_w);
    const int ty = r / p.tiles_w, tx = r % p.tiles_w;
    __syncthreads();
    if (aligned) {
      stem_stage_input(p, n, ty, tx, s_in);
      stem_stage_wait();
    } else {   // generic 2-byte path (odd image widths)
      const int iy0 = ty * kStemTH * 2 - 1, ixs = tx * kStemTW * 2 - 2;
      const __nv_bfloat16* img = p.x + (size_t)n * p.H * p.W * 3;
      for (int e = threadIdx.x; e < kStemIH * kStemSW * 3; e += 256) {
        const int rr = e / (kStemSW * 3), rem = e % (kStemSW * 3);
        const int iy = iy0 + rr, ix = ixs + rem / 3;
        __nv_bfloat16 v = __float2bfloat16(0.f);
        if ((unsigned)iy < (unsigned)p.H && (unsigned)ix < (unsigned)p.W)
          v = img[((size_t)iy * p.W + ix) * 3 + rem % 3];
        s_in[e] = v;
      }
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

// wgrad: thread = (8 output channels co8, 4 positions jq, pixel subset ps): 256 threads =
// (Cout/8) x 8 x PS.  32 FMAs per 2 + 4 shared-memory loads.  Positions are walked in
// staging order jj = (ky*3 + kx)*3 + ci and mapped to the parameter's j = ci*9 + ky*3 + kx at the end.
__global__ void __launch_bounds__(256) stem_wgrad_kernel(const __grid_constant__ StemDev p) {
  extern __shared__ __align__(16) unsigned char stem_smem[];
  __nv_bfloat16* s_in = reinterpret_cast<__nv_bfloat16*>(stem_smem);          // [IH][SW][3]
  __nv_bfloat16* s_dh = s_in + ((kStemIH * kStemSW * 3 + 7) & ~7);            // [TH*TW][Cout]
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
  const bool aligned = ((p.W * 3) % 2) == 0;
  for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
    const int n = t / (p.tiles_h * p.tiles_w), r = t % (p.tiles_h * p.tiles_w);
    const int ty = r / p.tiles_w, tx = r % p.tiles_w;
    __syncthreads();
    if (aligned) {
      stem_stage_input(p, n, ty, tx, s_in);
    } else {
      const int iy0 = ty * kStemTH * 2 - 1, ixs = tx * kStemTW * 2 - 2;
      const __nv_bfloat16* img = p.x + (size_t)n * p.H * p.W * 3;
      for (int e = threadIdx.x; e < kStemIH * kStemSW * 3; e += 256) {
        const int rr = e / (kStemSW * 3), rem = e % (kStemSW * 3);
        const int iy = iy0 + rr, ix = ixs + rem / 3;
        __nv_bfloat16 v = __float2bfloat16(0.f);
        if ((unsigned)iy < (unsigned)p.H && (unsigned)ix < (unsigned)p.W)
          v = img[((size_t)iy * p.W + ix) * 3 + rem % 3];
        s_in[e] = v;
      }
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
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(
                       smem_u32(reinterpret_cast<uint4*>(s_dh) + e)),
                   "l"(src), "r"(ok ? 16 : 0)
                   : "memory");
    }
    stem_stage_wait();
    __syncthreads();
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
static int stem_fill(const yamb_stem_conv* a, StemDev& p) {
  if (!a || a->N <= 0 || a->H <= 0 || a->W <= 0 || !a->x)
    return set_error(YAMB_EINVAL, "stem conv: bad arguments");
  if (a->Cout <= 0 || a->Cout > 64 || (a->Cout % 8))
    return set_error(YAMB_EINVAL, "stem conv: Cout=%d must be a multiple of 8, <= 64", a->Cout);
  p.N = a->N; p.H = a->H; p.W = a->W; p.Cout = a->Cout;
  p.Ho = (a->H - 1) / 2 + 1; p.Wo = (a->W - 1) / 2 + 1;
  p.x = (const __nv_bfloat16*)a->x; p.w = a->w; p.y = (__nv_bfloat16*)a->y;
  p.dh = (const __nv_bfloat16*)a->dh; p.dw = a->dw;
  p.tiles_h = (p.Ho + kStemTH - 1) / kStemTH;
  p.tiles_w = (p.Wo + kStemTW - 1) / kStemTW;
  long long nt = (long long)a->N * p.tiles_h * p.tiles_w;
  if (nt > 0x7fffffffLL) return set_error(YAMB_EINVAL, "stem conv: too many tiles");
  p.num_tiles = (int)nt;
  return 0;
}

template <bool EVAL>
static int stem_fwd_run(const StemDev& p, int Cout, cudaStream_t st) {
  const size_t smem = 27 * 64 * 4 + (size_t)((kStemIH * kStemSW * 3 + 7) & ~7) * 2 +
                      (size_t)8 * 64 * (Cout / 8) * 16;
  int per_sm = 0;
  const int rc = smem_optin("stem conv fwd", (const void*)stem_fwd_kernel<EVAL>, smem, &per_sm);
  if (rc) return rc;
  const int res_f = max_ctas() * (per_sm > 0 ? per_sm : 1);   // one resident wave: no tail
  stem_fwd_kernel<EVAL><<<p.num_tiles < res_f ? p.num_tiles : res_f, 256, smem, st>>>(p);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "stem conv fwd: %s", cudaGetErrorString(e));
  return 0;
}

int stem_conv_fwd_launch(const yamb_stem_conv* a, cudaStream_t st) {
  StemDev p;
  int rc = stem_fill(a, p);
  if (rc) return rc;
  if (!a->w || !a->y || (reinterpret_cast<uintptr_t>(a->y) & 15))
    return set_error(YAMB_EINVAL, "stem conv fwd: w / y (16-byte aligned) required");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  p.scale = p.shift = nullptr;
  p.act = 0;
  return stem_fwd_run<false>(p, a->Cout, st);
}

int stem_conv_eval_fwd_launch(const yamb_stem_conv_eval* a, cudaStream_t st) {
  if (!a) return set_error(YAMB_EINVAL, "stem conv eval: bad arguments");
  StemDev p;
  int rc = stem_fill(&a->conv, p);
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
  return stem_fwd_run<true>(p, a->conv.Cout, st);
}

int stem_conv_wgrad_launch(const yamb_stem_conv* a, cudaStream_t st) {
  StemDev p;
  int rc = stem_fill(a, p);
  if (rc) return rc;
  if (!a->dh || !a->dw || (reinterpret_cast<uintptr_t>(a->dh) & 15))
    return set_error(YAMB_EINVAL, "stem conv wgrad: dh (16-byte aligned) / dw required");
  if (256 % a->Cout) return set_error(YAMB_EINVAL, "stem conv wgrad: Cout must be 8, 16, 32 or 64");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  const size_t smem = (size_t)((kStemIH * kStemSW * 3 + 7) & ~7) * 2 +
                      (size_t)kStemTH * kStemTW * a->Cout * 2;
  // the grid sets the number of partial slabs and so the order of their sum: it comes from the
  // occupancy at this Cout's shared memory
  int per_sm = 0;
  if ((rc = smem_optin("stem conv wgrad", (const void*)stem_wgrad_kernel, smem, &per_sm))) return rc;
  const int res_w = max_ctas() * (per_sm > 0 ? per_sm : 1);
  const int grid = p.num_tiles < res_w ? p.num_tiles : res_w;
  const int slots = grid * (256 / p.Cout);
  rc = det_alloc((size_t)slots * p.Cout * 27 * sizeof(float), st, &p.part);
  if (rc) return rc;
  stem_wgrad_kernel<<<grid, 256, smem, st>>>(p);
  if (cudaPeekAtLastError() != cudaSuccess) det_free(p.part, st);
  else if ((rc = det_reduce_launch(p.part, slots, (long long)p.Cout * 27, p.dw, st)) != 0) return rc;
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "stem conv wgrad: %s", cudaGetErrorString(e));
  return 0;
}

}  // namespace yamb
