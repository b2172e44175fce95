// Eval-mode inverted-residual block in ONE launch, no intermediate tensor in HBM (sm_90a).
//
// Replaces, behind yamb_block_eval_fwd (include/yamb200.h), the whole forward of
// InvertedResidualChannels (reference models/mobilenet_base.py:446-451: 1x1 expand -> BatchNorm ->
// act -> depthwise 3x3 -> BatchNorm -> act -> 1x1 project -> BatchNorm (+x)) when every BatchNorm
// normalises with its running statistics (model.eval(): validation, utils/common.py forward_loss
// under torch.no_grad()).  With the statistics known up front the block is a pure function of an
// input tile plus a one-pixel halo: SURVEY.md §7.1 step 2 / §7.2, BASELINE.json's "fused block".
//
// Persistent CTAs (one per SM) walk output tiles of <= 112 pixels (k = 3, stride 1: 7x16, 7x14 or
// two 7x7 images; stride 2, k = 5 / 7 and wide outputs: smaller tiles) whose input tile with its
// halo fits 256 rows.  Per tile:
//   x tile (+halo, <= 256 pixels) --TMA 4-D box, zero fill outside the image--> smem (A operand)
//   for every 64-channel slice of the hidden dimension:
//     W1 slice --TMA--> smem
//     wgmma  [64 px x Cin] x [Cin x 64] per 64-pixel chunk -> registers (fp32)        expand
//     BatchNorm1 + act -> bf16, zero outside the image -> smem                         epilogue 1
//     kxk stencil on the CUDA cores -> BatchNorm2 + act -> bf16 -> smem (A operand layout)
//     W3 slice --TMA--> smem
//     wgmma  [64 px x 64] x [64 x 16 j]  accumulated over the slices -> registers      project
//   BatchNorm3 (+ x) -> bf16 -> global                                                 epilogue 2
// Blocks without the 1x1 expansion (hidden == input) skip the first MMA: the x panel itself is the
// stencil input.
// Squeeze-and-Excitation (InvertedResidualChannelsFused, reference mobilenet_base.py:336-339) is the
// MODE template flag: kGate multiplies a2 by gate[n][c] before the project; kPool (the pool pass,
// yamb_block_eval_pool_fwd) runs the same tile walk up to a2 and writes per-tile spatial means
// instead of the project (see the enum below).
// HBM traffic: x once (+ halo re-reads from L2), y once; the hidden tensors (6 x the block's
// input) never leave the SM.  BatchNorm folding (gamma * rsqrt(var + eps), beta - mean * scale) is
// done by the kernel from the module's own buffers: no preparation launches.
//
// Roles: 8 warps = two warpgroups.  Each warpgroup runs the expand MMAs and epilogue 1 of its
// 64-pixel chunks (chunks wg, wg + 2), and the project MMAs of its share of the output: the rows
// 64 wg.. of all columns when the tile has more than 64 pixels (Cout <= 160), else all rows of half
// of the 16-column groups — at most 80 fp32 accumulators per thread.  Warps 0-6 run the stencil
// (runs of 7 or 8 consecutive outputs of a row x 16 or 32 channel groups); one thread of warp 7
// issues the TMA loads.  Every staging buffer is single and refilled right after its last reader
// retired:
//   wait W1(c) | expand(c) -> epilogue 1 (the MMAs of project(c-1) retire here too) | S2 |
//   TMA W3(c), W1(c+1) [+ x of the next tile] || stencil -> a2 | S3 | project(c) (left in flight)
//
// Rounding points: a1 = bf16(act(bn1(fp32 accumulator))), a2 = bf16(act(bn2(fp32 stencil))),
// y = bf16(bn3(fp32 accumulator) + x) — one rounding fewer per stage than the four-launch path
// (which stores the raw convolution outputs in bf16 first); with the gate a2s = bf16(a2 * gate),
// pooled = fp32 mean of the bf16 a2.
//
// Cluster split (CLUSTER, yamb_block_eval_cluster_fwd / _pool_fwd; small batches, where a walk over
// the tiles leaves most SMs idle): the CS CTAs of a thread-block cluster take the same output tile
// and the contiguous slice ranges [r*NC/CS, (r+1)*NC/CS) of the hidden dimension.  Each runs the
// sequence above over its own slices; after the last one it stores its fp32 project accumulators
// in its own shared memory, and after a cluster barrier every rank adds the CS partials of its
// share of the output columns in rank order 0..CS-1 (DSMEM loads), then applies BatchNorm3 (+ x).
// The pool pass needs no exchange: each rank writes the pooled means of its own slices.
//
// block_eval.cu instantiates the unsplit kernels, block_eval_cluster.cu the cluster ones.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <string.h>

#include <map>
#include <mutex>
#include <tuple>

#include "host_util.h"
#include "prims.cuh"

namespace yamb {

struct BnEvalDev {
  const float *gamma, *beta, *mean, *var;
  float eps;
};

struct BlockEvalDev {
  int N, H, W, Ho, Wo, Cin, Chid, Cout, act, residual;
  const __nv_bfloat16* x;
  const float* wdw;
  BnEvalDev bn1, bn2, bn3;
  __nv_bfloat16* y;
  int tiles_h, tiles_w, num_tiles;
  int KB;            // 64-channel panels of the x tile / the W1 slice
  int nks;           // K steps (16 channels) of the expand MMA
  int Npad;          // Cout rounded up to a multiple of 16 (project MMAs of 16 columns)
  int NC;            // 64-channel slices of the hidden dimension
  int xpanel_bytes;  // bytes between the 64-channel panels of the x tile
  int off_w1, off_w3, off_h1, off_h2, off_tab, off_c3, off_bars;
  const float* gate; // kGate: [N][Chid] Squeeze-and-Excitation gate
  float* part;       // kPool: [tiles_h * tiles_w][N][Chid] per-tile partial means
  float inv_hw;      // kPool: 1 / (Ho * Wo)
  int mode;          // kPlain / kGate / kPool (host-side dispatch; the kernel has it as MODE)
  int cs;            // CLUSTER: CTAs per cluster (2, 4 or 8)
  int off_red;       // CLUSTER, not kPool: fp32 partials [NPO][red_pitch] of this CTA's slices
  int red_pitch;     // Npad + 8 (a quarter warp's rows on distinct banks) where that fits, else Npad
};

// What one launch computes:
//   kPlain  y = bn3(project(a2)) (+ x)
//   kGate   y = bn3(project(a2s)) (+ x),  a2s = bf16(a2 * gate[n][c])   (Squeeze-and-Excitation)
//   kPool   no project: every tile writes the spatial sums of a2 over its output pixels inside the
//           image, times 1 / (Ho * Wo), to its own slab of `part` (det_reduce adds the slabs)
enum { kPlain = 0, kGate = 1, kPool = 2 };

constexpr int kMaxProjChunks = 10;   // 16-column project accumulators per thread (80 registers)

constexpr int kH1Pitch = 144;    // bytes per pixel of the a1 tile: 64 bf16 + 16 (conflict-free, no swizzle)
// one set of per-slice tables: s1 t1 s2 t2 [64] + taps [K*K][64]
__host__ __device__ constexpr int tab_floats(int k) { return 256 + k * k * 64; }

// Output tile TI images x TOH x TOW pixels (<= 128: one or two 64-row project MMAs); the input tile
// with its halo is the M of the expand MMAs (NCH chunks of 64 rows, rows >= NPI are don't-care).
// Stencil threads (warps 0-6 = 224 threads): a thread owns CPT channels (64 / CPT channel groups)
// and RUN consecutive outputs of one output row.
template <int K_, int S_, int TOH_, int TOW_, int TI_, int CPT_>
struct EvGeom {
  static constexpr int K = K_, S = S_, TOH = TOH_, TOW = TOW_, TI = TI_, CPT = CPT_;
  static constexpr int P = (K - 1) / 2;
  static constexpr int IH = (TOH - 1) * S + K, IW = (TOW - 1) * S + K;
  static constexpr int NPI = TI * IH * IW;
  static constexpr int NPO = TI * TOH * TOW;
  static constexpr int RUN = (TOW % 8 == 0) ? 8 : 7;   // consecutive outputs of one row per stencil thread
  static constexpr int NRUN = NPO / RUN;
  static constexpr int NCG = 64 / CPT;                  // channel groups
  static constexpr int NCH = (NPI + 63) / 64;           // 64-row chunks of the expand MMAs
  static constexpr int PM = NPO > 64 ? 2 : 1;           // 64-row halves of the project MMAs
  static_assert(NPO <= 128 && NPI <= 256 && TOW % RUN == 0 && NRUN * NCG <= 224,
                "tile geometry (warp 7 must stay free of stencil work)");
};

template <class G, bool EXPAND, bool LEAN, int MODE, bool CLUSTER>
__global__ void __launch_bounds__(256, 1)
block_eval_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW1,
                  const __grid_constant__ CUtensorMap tmW3, const __grid_constant__ BlockEvalDev p) {
  constexpr bool POOL = MODE == kPool, GATE = MODE == kGate;
  constexpr int K = G::K, P = G::P, kTabFloats = tab_floats(G::K);
  constexpr int S = G::S, TOH = G::TOH, TOW = G::TOW, TI = G::TI, IH = G::IH, IW = G::IW;
  constexpr int NPI = G::NPI, NPO = G::NPO, RUN = G::RUN, NRUN = G::NRUN, CPT = G::CPT, NCG = G::NCG;
  constexpr int NCH = G::NCH, PM = G::PM;
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2, q = warp & 3;                              // warpgroup, warp inside it
  uint64_t* bar_ld = reinterpret_cast<uint64_t*>(smem + p.off_bars);  // TMA: W1 slice (+ x tile) landed
  uint64_t* bar_w3 = bar_ld + 1;                                       // TMA: W3 slice landed
  float* c3 = reinterpret_cast<float*>(smem + p.off_c3);     // [scale3 | shift3] x Npad
  float* tab = reinterpret_cast<float*>(smem + p.off_tab);   // two sets of kTabFloats
  uint8_t* sH1 = smem + p.off_h1;
  uint8_t* sH2 = smem + p.off_h2;
  const uint32_t sX_u = smem_u32(smem), sW1_u = sX_u + (uint32_t)p.off_w1,
                 sW3_u = sX_u + (uint32_t)p.off_w3, sH2_u = smem_u32(sH2);

  if (tid == 0) {
    mbar_init(bar_ld, 1);
    mbar_init(bar_w3, 1);
    fence_barrier_init();
  }
  for (int i = tid; i < (POOL ? 0 : p.Npad); i += 256) {
    float sc = 0.f, sh = 0.f;
    if (i < p.Cout) {
      const float r = rsqrtf(p.bn3.var[i] + p.bn3.eps);
      sc = (p.bn3.gamma ? p.bn3.gamma[i] : 1.f) * r;
      sh = (p.bn3.beta ? p.bn3.beta[i] : 0.f) - p.bn3.mean[i] * sc;
    }
    c3[i] = sc;
    c3[p.Npad + i] = sh;
  }
  // rows of the project A operand beyond the tile's pixels are never written: keep them zero
  for (int i = tid; i < 16384 / 16; i += 256) reinterpret_cast<uint4*>(sH2)[i] = make_uint4(0u, 0u, 0u, 0u);
  const bool control = warp == 7 && lane == 0;
  if (control) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmW1);
    if (!POOL) tma_prefetch_desc(&tmW3);
  }
  fence_proxy_async_smem();
  __syncthreads();
  const ActParam ap = make_act(p.act);
  constexpr bool lean = LEAN;       // relu / relu6 / none: clamp the packed bf16 pair
  const uint32_t lo2 = pack_bf16(ap.lo, ap.lo), hi2 = pack_bf16(ap.hi, ap.hi);

  // ---- per-slice coefficient tables (double-buffered), fetched one slice ahead into registers ----
  // threads 0..127: BatchNorm1 / BatchNorm2 of hidden channel slice*64 + tid%64;
  // thread (ch = tid/4, q = tid%4 < 3): taps 3q..3q+2 of that channel
  float pre_s = 0.f, pre_t = 0.f;
  // tab_fetch(c, tb): BatchNorm coefficients of slice c into registers (tab_store publishes them);
  // the K*K taps of its 64 channels go global -> tb by 4-byte cp.async (tid -> channel tid/4,
  // taps tid%4, tid%4 + 4, ...), complete before the S3 that precedes their first reader
  auto tab_fetch = [&](int c, float* tb) {
    if (tid < 128) {
      const BnEvalDev& b = tid < 64 ? p.bn1 : p.bn2;
      const int hc = c * 64 + (tid & 63);
      pre_s = pre_t = 0.f;
      if (hc < p.Chid && (EXPAND || tid >= 64)) {   // no expansion: there is no BatchNorm1
        const float r = rsqrtf(__ldg(b.var + hc) + b.eps);
        pre_s = (b.gamma ? __ldg(b.gamma + hc) : 1.f) * r;
        pre_t = (b.beta ? __ldg(b.beta + hc) : 0.f) - __ldg(b.mean + hc) * pre_s;
      }
    }
    const int ch = tid >> 2, hc = c * 64 + ch;
    const bool ok = hc < p.Chid;
    const float* src = p.wdw + (size_t)(ok ? hc : 0) * (K * K);
    const uint32_t dst = smem_u32(tb + 256 + ch);
#pragma unroll
    for (int tp = (tid & 3); tp < K * K; tp += 4)
      asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst + (uint32_t)(tp * 256)),
                   "l"(src + tp), "r"(ok ? 4 : 0) : "memory");
    cp_async_commit();
  };
  auto tab_store = [&](float* tb) {
    if (tid < 128) {
      const int which = tid >> 6, ch = tid & 63;
      tb[which * 128 + ch] = pre_s;          // s1 at 0, s2 at 128
      tb[which * 128 + 64 + ch] = pre_t;     // t1 at 64, t2 at 192
    }
    cp_async_wait<0>();   // this thread's taps have landed
  };

  // ---- TMA (control thread) ------------------------------------------------------------------------
  const int p_halves = p.Npad > 256 ? 2 : 1, p_nn = p.Npad / p_halves;
  uint32_t ld_par = 0, w3_par = 0;
  auto tma_x = [&](int t) {            // x tile of tile t: one 4-D box per 64-channel panel
    const int tx = t % p.tiles_w, ty = (t / p.tiles_w) % p.tiles_h, g = t / (p.tiles_w * p.tiles_h);
    for (int kb = 0; kb < p.KB; ++kb)
      tma_load_4d(&tmX, bar_ld, sX_u + (uint32_t)(kb * p.xpanel_bytes), kb * 64, tx * TOW * S - P,
                  ty * TOH * S - P, g * TI);
  };
  auto tma_w1 = [&](int c) {
    for (int kb = 0; kb < p.KB; ++kb)
      tma_load_2d(&tmW1, bar_ld, smem + p.off_w1 + kb * 8192, kb * 64, c * 64);
  };

  // ---- project MMAs of this warpgroup: rows p_row0.., 16-column groups [p_j0, p_j0 + p_nj) ----
  const int NJ = p.Npad >> 4;
  const int p_row0 = PM == 2 ? 64 * wg : 0;
  const int p_jh = PM == 2 ? NJ : (NJ + 1) / 2;
  const int p_j0 = PM == 2 ? 0 : wg * p_jh;
  const int p_nj = min(p_jh, NJ - p_j0);
  float pacc[kMaxProjChunks][8];

  // ---- per-thread geometry (the same in every tile) ------------------------------------------------
  // stencil: RUN consecutive outputs of one row x CPT channels
  const int cg = tid % NCG, sp = tid / NCG;
  const int r0 = sp * RUN;
  const int s_ti = r0 / (TOH * TOW), s_oy = (r0 % (TOH * TOW)) / TOW, s_ox0 = (r0 % (TOH * TOW)) % TOW;
  const uint8_t* s_hb = sH1 + (s_ti * IH * IW + s_oy * S * IW + s_ox0 * S) * kH1Pitch + cg * CPT * 2;

  // this CTA's slices [c_lo, c_hi) of every tile; the tiles of its cluster t0, t0 + t_step, ...
  const int cs = CLUSTER ? p.cs : 1;
  const int rank = CLUSTER ? (int)cluster_ctarank() : 0;
  const int c_lo = CLUSTER ? rank * p.NC / cs : 0, c_hi = CLUSTER ? (rank + 1) * p.NC / cs : p.NC;
  const int t_step = (int)gridDim.x / cs;
  int t = (int)blockIdx.x / cs;
  tab_fetch(c_lo, tab);
  tab_store(tab);
  if (control && t < p.num_tiles && (!CLUSTER || c_lo < c_hi)) {   // a rank may have no slice
    mbar_arrive_expect_tx(bar_ld, (uint32_t)(p.KB * (NPI * 128 + (EXPAND ? 8192 : 0))));
    tma_x(t);
    if (EXPAND) tma_w1(c_lo);
  }
  __syncthreads();   // tables of the first slice
  int gc = 0;
  for (; t < p.num_tiles; t += t_step) {
    const int tx = t % p.tiles_w, ty = (t / p.tiles_w) % p.tiles_h, g = t / (p.tiles_w * p.tiles_h);
    const bool more_tiles = t + t_step < p.num_tiles;
#pragma unroll
    for (int j = 0; j < kMaxProjChunks; ++j)
#pragma unroll
      for (int i = 0; i < 8; ++i) pacc[j][i] = 0.f;
    for (int c = c_lo; c < c_hi; ++c, ++gc) {
      const bool last_c = c + 1 == c_hi;
      const bool has_next = !last_c || more_tiles;
      const float* tb = tab + (gc & 1) * kTabFloats;
      if (EXPAND) {
        mbar_wait(bar_ld, ld_par);      // W1(c) (and the x tile) landed
        ld_par ^= 1;
#pragma unroll
        for (int mi = 0; mi < (NCH + 1) / 2; ++mi) {
          const int m = wg + 2 * mi;     // 64-pixel chunk of the input tile
          if (m >= NCH) break;
          float e[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) e[i] = 0.f;
          reg_fence(e);
          wgmma_fence();
#pragma unroll 1
          for (int ks = 0; ks < p.nks; ++ks) {
            const int kb = ks >> 2, kk = ks & 3;
            wgmma_m64n64<0, 0>(e, gmma_smem_desc(sX_u + (uint32_t)(kb * p.xpanel_bytes + m * 8192 + kk * 32), 16, 1024),
                               gmma_smem_desc(sW1_u + (uint32_t)(kb * 8192 + kk * 32), 16, 1024), 1u);
          }
          wgmma_commit();
          wgmma_wait<0>();               // (the previous slice's project MMAs retire here too)
          reg_fence(e);
          // ---- epilogue 1: a1 = bf16(act(bn1(h1))), zero outside the image, -> sH1[pixel][64] ----
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int r = m * 64 + q * 16 + (lane >> 2) + 8 * hh;
            if (r >= NPI) continue;
            const int ti = r / (IH * IW);
            const int dy = (r % (IH * IW)) / IW - P, dx = (r % (IH * IW)) % IW - P;
            const int n = g * TI + ti, yy = ty * TOH * S + dy, xx = tx * TOW * S + dx;
            const bool inside = n < p.N && (unsigned)yy < (unsigned)p.H && (unsigned)xx < (unsigned)p.W;
            uint8_t* dst = sH1 + r * kH1Pitch + (lane & 3) * 4;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int col = j * 8 + 2 * (lane & 3);
              const float2 ss = *reinterpret_cast<const float2*>(tb + col);
              const float2 tt = *reinterpret_cast<const float2*>(tb + 64 + col);
              const float2 v = ffma2(ss, make_float2(e[4 * j + 2 * hh], e[4 * j + 2 * hh + 1]), tt);
              uint32_t o;
              if (lean) {
                o = clamp_bf16x2(pack_bf16(v.x, v.y), lo2, hi2);
              } else {
                float a2[2] = {v.x, v.y};
                act_vec<2>(a2, ap);
                o = pack_bf16(a2[0], a2[1]);
              }
              *reinterpret_cast<uint32_t*>(dst + j * 16) = inside ? o : 0u;
            }
          }
        }
      } else {
        // ---- no expansion (hidden == input, reference mobilenet_base.py:397-404): the stencil input
        //      IS the x tile (already activated by its producer; TMA zero-filled the padding):
        //      panel c of the x tile -> sH1, un-swizzled ----
        if (c == c_lo) {
          mbar_wait(bar_ld, ld_par);    // every thread follows this barrier in the no-expand variant
          ld_par ^= 1;
        }
        if (tid < NPI) {
          const uint8_t* src = smem + c * p.xpanel_bytes + tid * 128;
          uint8_t* dst = sH1 + tid * kH1Pitch;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            *reinterpret_cast<uint4*>(dst + j * 16) =
                *reinterpret_cast<const uint4*>(src + ((j ^ (tid & 7)) << 4));
        }
        wgmma_wait<0>();                 // project(c-1) retired: sW3 and sH2 are free after S2
      }
      reg_fence(pacc);
      __syncthreads();                                                     // S2: a1 tile complete
      if (has_next) tab_fetch(last_c ? c_lo : c + 1, tab + ((gc + 1) & 1) * kTabFloats);
      if (warp == 7) {
        // ---- control: W3 slice in; the next slice's W1 (and the next tile's x) in ----
        if (lane == 0) {
          if (!POOL) {
            mbar_arrive_expect_tx(bar_w3, (uint32_t)(p.Npad * 128));
            for (int h = 0; h < p_halves; ++h)
              tma_load_2d(&tmW3, bar_w3, smem + p.off_w3 + h * p_nn * 128, c * 64, h * p_nn);
          }
          if (EXPAND) {
            if (has_next) {
              mbar_arrive_expect_tx(bar_ld, (uint32_t)(p.KB * (8192 + (last_c ? NPI * 128 : 0))));
              if (last_c) tma_x(t + t_step);
              tma_w1(last_c ? c_lo : c + 1);
            }
          } else if (last_c && more_tiles) {
            // every panel of this tile has been copied out: the next tile's x may land
            mbar_arrive_expect_tx(bar_ld, (uint32_t)(p.KB * NPI * 128));
            tma_x(t + t_step);
          }
        }
        __syncwarp();
      } else if (sp < NRUN) {
        // ---- KxK stencil: RUN consecutive outputs of one row x CPT channels per thread; the taps
        //      of one kernel row at a time in registers ----
        constexpr int NV = CPT / 2;          // fp32 pairs per pixel
        float2 o2[RUN][NV];
#pragma unroll
        for (int j = 0; j < RUN; ++j)
#pragma unroll
          for (int v = 0; v < NV; ++v) o2[j][v] = make_float2(0.f, 0.f);
#pragma unroll
        for (int ky = 0; ky < K; ++ky) {
          float2 w2[K][NV];
#pragma unroll
          for (int kx = 0; kx < K; ++kx) {
            const float* wp = tb + 256 + (ky * K + kx) * 64 + cg * CPT;
            if (CPT == 4) {
              const float4 wv = *reinterpret_cast<const float4*>(wp);
              w2[kx][0] = make_float2(wv.x, wv.y);
              w2[kx][NV - 1] = make_float2(wv.z, wv.w);
            } else {
              w2[kx][0] = *reinterpret_cast<const float2*>(wp);
            }
          }
#pragma unroll
          for (int ixx = 0; ixx < (RUN - 1) * S + K; ++ixx) {
            float2 av[NV];
            if (CPT == 4) {
              const uint2 a = *reinterpret_cast<const uint2*>(s_hb + (ky * IW + ixx) * kH1Pitch);
              av[0] = make_float2(bf16lo(a.x), bf16hi(a.x));
              av[NV - 1] = make_float2(bf16lo(a.y), bf16hi(a.y));
            } else {
              const uint32_t a = *reinterpret_cast<const uint32_t*>(s_hb + (ky * IW + ixx) * kH1Pitch);
              av[0] = make_float2(bf16lo(a), bf16hi(a));
            }
#pragma unroll
            for (int j = 0; j < RUN; ++j) {
              const int kx = ixx - j * S;   // compile-time after unrolling
              if (kx >= 0 && kx < K) {
#pragma unroll
                for (int v = 0; v < NV; ++v) o2[j][v] = ffma2(w2[kx][v], av[v], o2[j][v]);
              }
            }
          }
        }
        float2 s2v[NV], t2v[NV];
#pragma unroll
        for (int v = 0; v < NV; ++v) {
          s2v[v] = *reinterpret_cast<const float2*>(tb + 128 + cg * CPT + 2 * v);
          t2v[v] = *reinterpret_cast<const float2*>(tb + 192 + cg * CPT + 2 * v);
        }
        // the image of this run's outputs (TI = 2: the second image of the last tile may be past N)
        const int s_n = g * TI + s_ti;
        float2 gv[NV];                       // kGate: gate of this run's image, 0 past N / Chid
        if (GATE) {
          const int hc = c * 64 + cg * CPT;  // CPT | 8 | Chid: all CPT channels in range, or none
          const bool ok = s_n < p.N && hc < p.Chid;
#pragma unroll
          for (int v = 0; v < NV; ++v)
            gv[v] = ok ? make_float2(__ldg(p.gate + (size_t)s_n * p.Chid + hc + 2 * v),
                                     __ldg(p.gate + (size_t)s_n * p.Chid + hc + 2 * v + 1))
                       : make_float2(0.f, 0.f);
        }
        float2 ps[NV];                       // kPool: sums of a2 over this run's outputs in the image
#pragma unroll
        for (int v = 0; v < NV; ++v) ps[v] = make_float2(0.f, 0.f);
        const int boff = cg * CPT * 2;       // byte offset of this thread's channels inside a row
#pragma unroll
        for (int j = 0; j < RUN; ++j) {
          uint32_t wv[NV];
#pragma unroll
          for (int v = 0; v < NV; ++v) {
            const float2 z = ffma2(s2v[v], o2[j][v], t2v[v]);
            if (lean) {
              wv[v] = clamp_bf16x2(pack_bf16(z.x, z.y), lo2, hi2);
            } else {
              float qq[2] = {z.x, z.y};
              act_vec<2>(qq, ap);
              wv[v] = pack_bf16(qq[0], qq[1]);
            }
            if (GATE) wv[v] = pack_bf16(bf16lo(wv[v]) * gv[v].x, bf16hi(wv[v]) * gv[v].y);
          }
          if (POOL) {
            const bool in = s_n < p.N && ty * TOH + s_oy < p.Ho && tx * TOW + s_ox0 + j < p.Wo;
#pragma unroll
            for (int v = 0; v < NV; ++v)
              if (in) ps[v] = make_float2(ps[v].x + bf16lo(wv[v]), ps[v].y + bf16hi(wv[v]));
          } else {
            const int r = r0 + j;
            uint8_t* dst = sH2 + r * 128 + (((boff >> 4) ^ (r & 7)) << 4) + (boff & 15);
            if (CPT == 4) *reinterpret_cast<uint2*>(dst) = make_uint2(wv[0], wv[NV - 1]);
            else *reinterpret_cast<uint32_t*>(dst) = wv[0];
          }
        }
        if (POOL) {   // -> red[sp][channel] (the sH2 buffer, unused without the project MMAs)
#pragma unroll
          for (int v = 0; v < NV; ++v)
            *reinterpret_cast<float2*>(reinterpret_cast<float*>(sH2) + sp * 64 + cg * CPT + 2 * v) = ps[v];
        }
      }
      if (has_next) tab_store(tab + ((gc + 1) & 1) * kTabFloats);   // its readers are behind S3
      fence_proxy_async_smem();
      __syncthreads();                                                     // S3: a2 tile complete
      if (POOL) {
        // ---- pool: per (image, channel) of the slice, the stencil threads' sums in run order ->
        //      this tile's slab; red is rewritten only after the next S2 ----
        constexpr int RPI = TOH * TOW / RUN;     // runs per image
        if (tid < TI * 64) {
          const int ti = tid >> 6, ch = tid & 63;
          const float* red = reinterpret_cast<const float*>(sH2);
          float s = 0.f;
#pragma unroll 1
          for (int r = ti * RPI; r < (ti + 1) * RPI; ++r) s += red[r * 64 + ch];
          const int n = g * TI + ti, hc = c * 64 + ch;
          if (n < p.N && hc < p.Chid)
            p.part[((size_t)(ty * p.tiles_w + tx) * p.N + n) * p.Chid + hc] = s * p.inv_hw;
        }
        continue;
      }
      // ---- project(c): [64 px x 64] x [64 x 16 j], accumulated over the slices, left in flight ----
      mbar_wait(bar_w3, w3_par);       // landed during the stencil
      w3_par ^= 1;
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < kMaxProjChunks; ++j) {
        if (j >= p_nj) break;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          wgmma_m64n16<0, 0>(pacc[j], gmma_smem_desc(sH2_u + (uint32_t)(p_row0 * 128 + kk * 32), 16, 1024),
                             gmma_smem_desc(sW3_u + (uint32_t)((p_j0 + j) * 2048 + kk * 32), 16, 1024), 1u);
      }
      wgmma_commit();
    }
    if (POOL) continue;
    // ---- epilogue 2: y = bf16(bn3(h3) (+ x)) ----
    wgmma_wait<0>();
    reg_fence(pacc);
    auto store_y = [&](size_t pix, int col, float h0, float h1) {
      float v0 = fmaf(c3[col], h0, c3[p.Npad + col]);
      float v1 = fmaf(c3[col + 1], h1, c3[p.Npad + col + 1]);
      if (p.residual) {
        const uint32_t rx = __ldg(reinterpret_cast<const uint32_t*>(p.x + pix * p.Cin + col));
        v0 += bf16lo(rx);
        v1 += bf16hi(rx);
      }
      *reinterpret_cast<uint32_t*>(p.y + pix * p.Cout + col) = pack_bf16(v0, v1);
    };
    if (CLUSTER) {
      // ---- this CTA's partials -> red[row][col] (own shared memory, rows < NPO) ----
      const int rp = p.red_pitch;
      float* red = reinterpret_cast<float*>(smem + p.off_red);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = p_row0 + q * 16 + (lane >> 2) + 8 * hh;
        if (r >= NPO) continue;
#pragma unroll
        for (int j = 0; j < kMaxProjChunks; ++j) {
          if (j >= p_nj) break;
#pragma unroll
          for (int h8 = 0; h8 < 2; ++h8)
            *reinterpret_cast<float2*>(red + r * rp + (p_j0 + j) * 16 + h8 * 8 + 2 * (lane & 3)) =
                make_float2(pacc[j][4 * h8 + 2 * hh], pacc[j][4 * h8 + 2 * hh + 1]);
        }
      }
      cluster_sync();   // every rank's partials of this tile are in place
      // ---- column pairs [lo, hi) of every row: the cs partials in rank order, BatchNorm3 (+ x) ----
      const int npair = p.Cout >> 1, lo = rank * npair / cs, nw = (rank + 1) * npair / cs - lo;
      const uint32_t red_u = smem_u32(red);
      for (int i = tid; i < NPO * nw; i += 256) {
        const int r = i / nw, col = 2 * (lo + i % nw);
        const int ti = r / (TOH * TOW);
        const int oy = (r % (TOH * TOW)) / TOW, ox = (r % (TOH * TOW)) % TOW;
        const int n = g * TI + ti, yy = ty * TOH + oy, xx = tx * TOW + ox;
        if (!(n < p.N && yy < p.Ho && xx < p.Wo)) continue;
        const size_t pix = (size_t)(n * p.Ho + yy) * p.Wo + xx;
        const uint32_t a = red_u + (uint32_t)((r * rp + col) * 4);
        float2 part[8];
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if (k < cs) part[k] = dsmem_ld_f2(dsmem_map(a, (uint32_t)k));
        float2 s = part[0];
#pragma unroll
        for (int k = 1; k < 8; ++k)
          if (k < cs) s = make_float2(s.x + part[k].x, s.y + part[k].y);
        store_y(pix, col, s.x, s.y);
      }
      cluster_sync();   // the peers have read this CTA's partials: red may be rewritten
    } else {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = p_row0 + q * 16 + (lane >> 2) + 8 * hh;
        const int ti = r / (TOH * TOW);
        const int oy = (r % (TOH * TOW)) / TOW, ox = (r % (TOH * TOW)) % TOW;
        const int n = g * TI + ti, yy = ty * TOH + oy, xx = tx * TOW + ox;
        if (!(r < NPO && n < p.N && yy < p.Ho && xx < p.Wo)) continue;
        const size_t pix = (size_t)(n * p.Ho + yy) * p.Wo + xx;
#pragma unroll
        for (int j = 0; j < kMaxProjChunks; ++j) {
          if (j >= p_nj) break;
#pragma unroll
          for (int h8 = 0; h8 < 2; ++h8) {
            const int col = (p_j0 + j) * 16 + h8 * 8 + 2 * (lane & 3);
            if (col >= p.Cout) continue;
            store_y(pix, col, pacc[j][4 * h8 + 2 * hh], pacc[j][4 * h8 + 2 * hh + 1]);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
static int make_map(CUtensorMap* map, const void* ptr, int rank, const cuuint64_t* dims,
                    const cuuint64_t* strides_bytes, const cuuint32_t* box) {
  static PFN_encodeTiled encode = get_encode_tiled();
  if (!encode) return set_error(YAMB_ECUDA, "cuTensorMapEncodeTiled entry point not found");
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr),
                      dims, strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(YAMB_ECUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return 0;
}

// a launch of `grid` CTAs of 256 threads in clusters of `cs` along x; attr: one entry
static void cluster_launch_config(cudaLaunchConfig_t* cfg, cudaLaunchAttribute* attr, int grid, int smem,
                                  int cs, cudaStream_t st) {
  cfg->gridDim = dim3((unsigned)grid);
  cfg->blockDim = dim3(256);
  cfg->dynamicSmemBytes = (size_t)smem;
  cfg->stream = st;
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)cs;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg->attrs = attr;
  cfg->numAttrs = 1;
}

// clusters of `cs` CTAs of `kern` at `smem` bytes the current device holds at once (cached per
// kernel, device, smem and cs)
static int max_active_clusters(const void* kern, int smem, int cs, long long* out) {
  static std::mutex mu;
  static std::map<std::tuple<const void*, int, int, int>, int> cache;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "block_eval: %s", cudaGetErrorString(e));
  std::lock_guard<std::mutex> lock(mu);
  const auto key = std::make_tuple(kern, dev, smem, cs);
  auto it = cache.find(key);
  if (it == cache.end()) {
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    cluster_launch_config(&cfg, attr, cs, smem, cs, 0);
    int n = 0;
    e = cudaOccupancyMaxActiveClusters(&n, kern, &cfg);
    if (e != cudaSuccess) {
      cudaGetLastError();
      return set_error(YAMB_ECUDA, "block_eval: cluster occupancy: %s", cudaGetErrorString(e));
    }
    it = cache.emplace(key, n).first;
  }
  if (it->second <= 0)
    return set_error(YAMB_EINVAL, "block_eval: no cluster of %d CTAs with %d B of shared memory fits", cs, smem);
  *out = it->second;
  return 0;
}

template <class G, bool EXPAND, bool LEAN, int MODE, bool CLUSTER>
static int launch_eval_act(BlockEvalDev& p, const yamb_block_eval* a, cudaStream_t st) {
  // ---- shared-memory plan (bytes from the 1024-aligned base) ----
  // x tile: NPI rows of 128 B per 64-channel panel; the last 64-row MMA chunk of a panel reads
  // past them (rows that are never used): those reads stay inside this CTA's allocation
  p.xpanel_bytes = (G::NPI * 128 + 1023) & ~1023;
  int off = p.KB * p.xpanel_bytes;
  p.off_w1 = off; off += EXPAND ? p.KB * 8192 : 0;
  p.off_w3 = off; off += p.Npad * 128;
  p.off_h2 = (off + 1023) & ~1023; off = p.off_h2 + 16384;
  p.off_h1 = off; off += ((G::NPI * kH1Pitch) + 15) & ~15;
  p.off_tab = off; off += 2 * tab_floats(G::K) * 4;
  p.off_c3 = off; off += 2 * p.Npad * 4;
  p.off_bars = (off + 15) & ~15; off = p.off_bars + 16;
  if (CLUSTER && MODE != kPool) {   // the partials the cluster exchanges: NPO rows
    p.off_red = (off + 15) & ~15;
    p.red_pitch = p.off_red + G::NPO * (p.Npad + 8) * 4 <= 227 * 1024 ? p.Npad + 8 : p.Npad;
    off = p.off_red + G::NPO * p.red_pitch * 4;
  }
  int smem = off;
  const int x_read_end = (p.KB - 1) * p.xpanel_bytes + G::NCH * 8192;   // last byte the expand MMA may touch
  if (smem < x_read_end) smem = x_read_end;
  if (smem > 227 * 1024) return set_error(YAMB_EINVAL, "block_eval: tile does not fit shared memory");
  // project accumulators per thread: 64 x Npad (one 64-row half) or half of the 16-column groups
  const int chunks = G::PM == 2 ? p.Npad / 16 : (p.Npad / 16 + 1) / 2;
  if (chunks > kMaxProjChunks) return set_error(YAMB_EINVAL, "block_eval: accumulators exceed the registers");
  const int groups = (p.N + G::TI - 1) / G::TI;
  p.tiles_h = (p.Ho + G::TOH - 1) / G::TOH;
  p.tiles_w = (p.Wo + G::TOW - 1) / G::TOW;
  if ((long long)groups * p.tiles_h * p.tiles_w > 0x7fffffffLL)
    return set_error(YAMB_EINVAL, "block_eval: too many tiles");
  p.num_tiles = groups * p.tiles_h * p.tiles_w;
  // ---- tensor maps: x [N][H][W][Cin] (4-D box with halo), W1 [Chid][Cin], W3 [Cout][Chid] ----
  CUtensorMap tmX, tmW1, tmW3;
  {
    const cuuint64_t dims[4] = {(cuuint64_t)p.Cin, (cuuint64_t)p.W, (cuuint64_t)p.H, (cuuint64_t)p.N};
    const cuuint64_t str[3] = {(cuuint64_t)p.Cin * 2, (cuuint64_t)p.W * p.Cin * 2,
                               (cuuint64_t)p.H * p.W * p.Cin * 2};
    const cuuint32_t box[4] = {64, (cuuint32_t)G::IW, (cuuint32_t)G::IH, (cuuint32_t)G::TI};
    int rc = make_map(&tmX, a->x, 4, dims, str, box);
    if (rc) return rc;
  }
  memset(&tmW1, 0, sizeof(tmW1));
  memset(&tmW3, 0, sizeof(tmW3));
  if (EXPAND) {
    const cuuint64_t dims[2] = {(cuuint64_t)p.Cin, (cuuint64_t)p.Chid};
    const cuuint64_t str[1] = {(cuuint64_t)p.Cin * 2};
    const cuuint32_t box[2] = {64, 64};
    int rc = make_map(&tmW1, a->w_expand, 2, dims, str, box);
    if (rc) return rc;
  }
  if (MODE != kPool) {
    const int halves = p.Npad > 256 ? 2 : 1;
    const cuuint64_t dims[2] = {(cuuint64_t)p.Chid, (cuuint64_t)p.Cout};
    const cuuint64_t str[1] = {(cuuint64_t)p.Chid * 2};
    const cuuint32_t box[2] = {64, (cuuint32_t)(p.Npad / halves)};
    int rc = make_map(&tmW3, a->w_project, 2, dims, str, box);
    if (rc) return rc;
  }
  const void* kern = (const void*)block_eval_kernel<G, EXPAND, LEAN, MODE, CLUSTER>;
  int rc = smem_optin("block_eval", kern, smem, nullptr, 256, /*max_carveout=*/true);
  if (rc) return rc;
  // One resident CTA per SM: the project accumulators, the stencil and the expand fragments take
  // more than the 128 registers per thread that two CTAs of 256 threads could have.  Clusters: at
  // most one cluster per tile and no more than the device holds at once.
  long long cap = (long long)max_ctas();
  if (CLUSTER && (rc = max_active_clusters(kern, smem, p.cs, &cap))) return rc;
  const int grid = (int)(p.num_tiles < cap ? p.num_tiles : cap) * (CLUSTER ? p.cs : 1);
  auto run = [&]() -> cudaError_t {
    if (!CLUSTER) {
      block_eval_kernel<G, EXPAND, LEAN, MODE, CLUSTER><<<grid, 256, smem, st>>>(tmX, tmW1, tmW3, p);
      return cudaGetLastError();
    }
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    cluster_launch_config(&cfg, attr, grid, smem, p.cs, st);
    return cudaLaunchKernelEx(&cfg, block_eval_kernel<G, EXPAND, LEAN, MODE, CLUSTER>, tmX, tmW1, tmW3, p);
  };
  if (MODE != kPool) {
    cudaError_t e = run();
    if (e != cudaSuccess) return set_error(YAMB_ECUDA, "block_eval launch: %s", cudaGetErrorString(e));
    return 0;
  }
  // pool pass: one slab of N x Chid partial means per spatial tile position, every element
  // written by exactly one tile; pooled = 0, then += the slabs in slab order (deterministic)
  const int nslab = p.tiles_h * p.tiles_w;
  const long long n_out = (long long)p.N * p.Chid;
  if ((rc = det_alloc((size_t)nslab * n_out * sizeof(float), st, &p.part))) return rc;
  p.inv_hw = 1.f / ((float)p.Ho * (float)p.Wo);
  cudaError_t e = cudaMemsetAsync(a->pooled, 0, (size_t)n_out * sizeof(float), st);
  if (e == cudaSuccess) e = run();
  if (e != cudaSuccess) {
    det_free(p.part, st);
    return set_error(YAMB_ECUDA, "block_eval pool launch: %s", cudaGetErrorString(e));
  }
  return det_reduce_launch(p.part, nslab, n_out, a->pooled, st);
}

template <class G, bool EXPAND, int MODE, bool CLUSTER>
static int launch_eval_mode(BlockEvalDev& p, const yamb_block_eval* a, cudaStream_t st) {
  // relu / relu6 / none are clamps of the packed bf16 pair; swish / h-swish take the generic path
  const bool lean = a->act == YAMB_ACT_NONE || a->act == YAMB_ACT_RELU || a->act == YAMB_ACT_RELU6;
  return lean ? launch_eval_act<G, EXPAND, true, MODE, CLUSTER>(p, a, st)
              : launch_eval_act<G, EXPAND, false, MODE, CLUSTER>(p, a, st);
}

template <class G, bool EXPAND, bool CLUSTER>
static int launch_eval(BlockEvalDev& p, const yamb_block_eval* a, cudaStream_t st) {
  if (p.mode == kPool) return launch_eval_mode<G, EXPAND, kPool, CLUSTER>(p, a, st);
  if (p.mode == kGate) return launch_eval_mode<G, EXPAND, kGate, CLUSTER>(p, a, st);
  return launch_eval_mode<G, EXPAND, kPlain, CLUSTER>(p, a, st);
}

// CLUSTER: the hidden slices of every tile split over clusters of `cs` CTAs (2, 4 or 8); else cs = 1
template <bool CLUSTER>
static int block_eval_launch_impl(const yamb_block_eval* a, cudaStream_t st, bool pool, int cs) {
  if (!a) return set_error(YAMB_EINVAL, "null args");
  if (CLUSTER ? (cs != 2 && cs != 4 && cs != 8) : cs != 1)
    return set_error(YAMB_EINVAL, "block_eval: cluster size must be 2, 4 or 8 (got %d)", cs);
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  if (a->N <= 0 || a->H <= 0 || a->W <= 0) return set_error(YAMB_EINVAL, "block_eval: bad shape");
  if (a->Cin % 8 || a->Chid % 8 || a->Cout % 8 || a->Cin <= 0 || a->Chid <= 0 || a->Cout <= 0)
    return set_error(YAMB_EINVAL, "block_eval: channel counts must be positive multiples of 8");
  if (a->Cin > 256 || a->Cout > 320)
    return set_error(YAMB_EINVAL, "block_eval: Cin <= 256, Cout <= 320 (got %d, %d)", a->Cin, a->Cout);
  if ((a->kernel != 3 && a->kernel != 5 && a->kernel != 7) || (a->stride != 1 && a->stride != 2))
    return set_error(YAMB_EINVAL, "block_eval: depthwise k in {3,5,7}, stride 1 or 2 (got k=%d s=%d)",
                     a->kernel, a->stride);
  if (a->kernel != 3 && !a->w_expand)
    return set_error(YAMB_EINVAL, "block_eval: k = 5 / 7 is built with expansion only");
  if (!a->w_expand && a->Chid != a->Cin)
    return set_error(YAMB_EINVAL, "block_eval: no expand weights needs Chid == Cin");
  if (a->residual && a->stride != 1)
    return set_error(YAMB_EINVAL, "block_eval: residual needs stride 1");
  if (a->residual && a->Cin != a->Cout)
    return set_error(YAMB_EINVAL, "block_eval: residual needs Cin == Cout");
  // the pool pass reads x, W1, the depthwise weights and BatchNorms 1 / 2 and writes `pooled`
  if (!a->x || !a->w_dw || (pool ? !a->pooled : (!a->y || !a->w_project)))
    return set_error(YAMB_EINVAL, "block_eval: null pointer");
  const yamb_bn_eval* bns[3] = {&a->bn1, &a->bn2, &a->bn3};
  for (int i = a->w_expand ? 0 : 1; i < (pool ? 2 : 3); ++i)
    if (!bns[i]->running_mean || !bns[i]->running_var)
      return set_error(YAMB_EINVAL, "block_eval: BatchNorm %d has no running statistics", i + 1);
  if ((((uintptr_t)a->x) | ((uintptr_t)a->y) | ((uintptr_t)a->w_expand) | ((uintptr_t)a->w_project)) & 15)
    return set_error(YAMB_EINVAL, "block_eval: tensors must be 16-byte aligned");
  if (!pool && a->gate && ((uintptr_t)a->gate & 7))
    return set_error(YAMB_EINVAL, "block_eval: gate must be 8-byte aligned");
  if ((long long)a->N * a->H * a->W > 0x7fffffffLL / 2)
    return set_error(YAMB_EINVAL, "block_eval: too many pixels");
  BlockEvalDev p;
  memset(&p, 0, sizeof(p));
  p.N = a->N; p.H = a->H; p.W = a->W;
  p.Ho = (a->H - 1) / a->stride + 1;      // pad 1, k 3
  p.Wo = (a->W - 1) / a->stride + 1;
  p.Cin = a->Cin; p.Chid = a->Chid; p.Cout = a->Cout;
  p.act = a->act; p.residual = a->residual ? 1 : 0;
  p.x = (const __nv_bfloat16*)a->x; p.y = (__nv_bfloat16*)a->y;
  p.wdw = a->w_dw;
  p.gate = a->gate;
  p.mode = pool ? kPool : (a->gate ? kGate : kPlain);
  p.cs = cs;
  auto cvt = [](const yamb_bn_eval& s) {
    BnEvalDev d;
    d.gamma = s.gamma; d.beta = s.beta; d.mean = s.running_mean; d.var = s.running_var; d.eps = s.eps;
    return d;
  };
  p.bn1 = cvt(a->bn1); p.bn2 = cvt(a->bn2); p.bn3 = cvt(a->bn3);
  const int kpad = (a->Cin + 15) / 16 * 16;
  p.nks = kpad / 16;
  p.KB = (kpad + 63) / 64;
  p.Npad = (a->Cout + 15) / 16 * 16;
  p.NC = (a->Chid + 63) / 64;
  const bool ex = a->w_expand != nullptr;
  // fewest tiles among the geometries of (k, stride); each holds its input tile in <= 256 rows.
  // Tiles of more than 64 output pixels keep 64 x Npad project accumulators per thread: wide
  // outputs (Npad > 160) take one 7x7 image per tile instead.
  const bool wide = p.Npad > 16 * kMaxProjChunks;
  auto tiles_of = [&](int toh, int tow, int ti) {
    return (long long)((p.Ho + toh - 1) / toh) * ((p.Wo + tow - 1) / tow) * ((a->N + ti - 1) / ti);
  };
  if (a->kernel == 3) {
    if (a->stride == 2)   // 7x7 outputs from a 15x15 input tile, 2 channels per stencil thread
      return ex ? launch_eval<EvGeom<3, 2, 7, 7, 1, 2>, true, CLUSTER>(p, a, st)
                : launch_eval<EvGeom<3, 2, 7, 7, 1, 2>, false, CLUSTER>(p, a, st);
    if (wide)
      return ex ? launch_eval<EvGeom<3, 1, 7, 7, 1, 4>, true, CLUSTER>(p, a, st)
                : launch_eval<EvGeom<3, 1, 7, 7, 1, 4>, false, CLUSTER>(p, a, st);
    const long long t0 = tiles_of(7, 16, 1), t1 = tiles_of(7, 14, 1), t2 = tiles_of(7, 7, 2);
    if (t0 <= t1 && t0 <= t2)
      return ex ? launch_eval<EvGeom<3, 1, 7, 16, 1, 4>, true, CLUSTER>(p, a, st)
                : launch_eval<EvGeom<3, 1, 7, 16, 1, 4>, false, CLUSTER>(p, a, st);
    if (t1 <= t2)
      return ex ? launch_eval<EvGeom<3, 1, 7, 14, 1, 4>, true, CLUSTER>(p, a, st)
                : launch_eval<EvGeom<3, 1, 7, 14, 1, 4>, false, CLUSTER>(p, a, st);
    return ex ? launch_eval<EvGeom<3, 1, 7, 7, 2, 4>, true, CLUSTER>(p, a, st)
              : launch_eval<EvGeom<3, 1, 7, 7, 2, 4>, false, CLUSTER>(p, a, st);
  }
  if (a->kernel == 5) {
    if (a->stride == 2) return launch_eval<EvGeom<5, 2, 6, 7, 1, 2>, true, CLUSTER>(p, a, st);
    if (wide) return launch_eval<EvGeom<5, 1, 7, 7, 1, 4>, true, CLUSTER>(p, a, st);
    const long long t0 = tiles_of(7, 16, 1), t1 = tiles_of(7, 14, 1), t2 = tiles_of(7, 7, 2);
    if (t0 <= t1 && t0 <= t2) return launch_eval<EvGeom<5, 1, 7, 16, 1, 4>, true, CLUSTER>(p, a, st);
    if (t1 <= t2) return launch_eval<EvGeom<5, 1, 7, 14, 1, 4>, true, CLUSTER>(p, a, st);
    return launch_eval<EvGeom<5, 1, 7, 7, 2, 4>, true, CLUSTER>(p, a, st);
  }
  if (a->stride == 2) return launch_eval<EvGeom<7, 2, 4, 7, 1, 2>, true, CLUSTER>(p, a, st);
  return launch_eval<EvGeom<7, 1, 7, 7, 1, 2>, true, CLUSTER>(p, a, st);
}

}  // namespace yamb
