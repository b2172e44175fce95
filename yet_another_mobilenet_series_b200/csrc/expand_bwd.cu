// Expand-side backward of an inverted-residual block in one pass (sm_90a):
//
//   dh1 = ca1 * dz1 + cb1 * h1 + cc1          (BatchNorm-1 backward, formed once per element)
//   dx  = dh1 * W1 (+ dy)                     [M][Cin]   bf16
//   dW1 += dh1^T * x                          [Chid][Cin] fp32
//
// The two 1x1-convolution gradients of the expand conv read the same Chid-wide tensors dz1 and h1.
// As two GEMMs (yamb_pointwise_gemm dgrad + split-K wgrad) each one streams them from HBM and forms
// dh1 in its own loaders; here one persistent kernel reads them once.  In SWIZZLE_128B a staged
// [128 px x 64 ch] dh1 panel is at the same time the K-major A k-block of the dgrad and the MN-major
// A m64 block of the wgrad, so both products are issued on the same shared-memory bytes.
//
// One CTA (384 threads) per SM, warp-specialised:
//   warp 0      TMA producer: dz1 and h1 panels [128 px x 64 ch] into a ring of stages
//   warps 4-7   one consumer warpgroup: per panel 2 x 4 dgrad wgmmas (dx of the unit) and 8
//               wgrad wgmmas (dW1 rows of the panel, held in registers over the slab); dx
//               epilogue (+ residual) per unit, the slab's dW1 partial at the end of each slab
//   warps 8-11  rewrite each landed panel in place into dh1 (the GEMM loaders' two-source
//               transform, same expression and rounding) and bring the unit's x rows by cp.async
// The work is the split-K wgrad GEMM's: its slabs of consecutive pixels (yamb_gemm_plan of that
// wgrad), each walked in 128-pixel units from its first pixel, one dW1 partial per slab accumulated
// in the same k16 order from zero.  det_reduce_launch adds the slabs into dW1 in slab order as the
// GEMM's split-K reduction does, so dW1 is bitwise the two-GEMM path's; `+=` so that gradient
// accumulation over micro-batches works.  dx rows are independent of the walk.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <string.h>

#include "host_util.h"
#include "prims.cuh"

namespace yamb {

constexpr int kXbRows = 128;                   // pixels per unit of a slab's walk
constexpr int kXbPanel = kXbRows * 128;        // one [128 px x 64 ch] bf16 panel, 16 KB
constexpr int kXbStage = 2 * kXbPanel;         // dz1 panel (rewritten to dh1) + h1 panel
constexpr int kXbWPanel = 64 * 128;            // W1 rows of one panel: [64 ch][64 (Cin, padded)]
constexpr int kXbMaxStages = 6;
constexpr int kXbMaxPanels = 3;                // Chid <= 192
constexpr int kXbThreads = 384;

struct XbBars {
  uint64_t tma_full[kXbMaxStages];   // the TMA landed dz1 / h1 of the stage
  uint64_t full[kXbMaxStages];       // dh1 of the stage formed (and the x rows of its unit)
  uint64_t empty[kXbMaxStages];      // the consumer's wgmmas that read the stage retired
  uint64_t x_empty[2];               // the x tile buffer may be overwritten
};

struct XbDev {
  int M, Cin, Chid, panels, num_stages;
  int slabs, slab_rows;              // the split-K wgrad's slabs: slab s = pixels [s, s + 1) * slab_rows
  const float *ca, *cb, *cc;
  const __nv_bfloat16 *W1, *x, *residual;
  __nv_bfloat16* dx;
  float* part;                       // [slabs][Chid][Cin] per-slab dW1 partials
  int off_x, off_w, off_bars;        // shared-memory offsets (bytes) of the x ring, W1, barriers
};

// Bounded wait without a call in it (a call between wgmma issue and wait serialises the wgmmas).
__device__ __forceinline__ void xb_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = global_timer_ns();
  while (!mbar_try_wait(bar, parity))
    if (global_timer_ns() - t0 > 4000000000ull) __trap();
}

template <int TA, int TB, int BN>
__device__ __forceinline__ void xb_mma(float (&d)[BN / 2], uint64_t da, uint64_t db) {
  if constexpr (BN == 32) wgmma_m64n32<TA, TB>(d, da, db, 1u);
  else wgmma_m64n16<TA, TB>(d, da, db, 1u);
}

// kBN: wgmma width (Cin padded to 16 or 32); kNP: 64-channel panels of Chid.  Both compile-time so
// that the consumer's wgmma sequence is straight-line code (a branch around a wgmma makes ptxas
// serialise all of them).
template <int kBN, int kNP>
__global__ void __launch_bounds__(kXbThreads, 1)
expand_bwd_kernel(const __grid_constant__ CUtensorMap tmDz, const __grid_constant__ CUtensorMap tmH,
                  const __grid_constant__ XbDev p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  XbBars* bars = reinterpret_cast<XbBars*>(smem + p.off_bars);
  const uint32_t s_stage = smem_u32(smem);
  const uint32_t s_x = smem_u32(smem + p.off_x);
  const uint32_t s_w = smem_u32(smem + p.off_w);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = p.num_stages;

  if (threadIdx.x == 32) {
    for (int i = 0; i < S; ++i) {
      mbar_init(&bars->tma_full[i], 1);
      mbar_init(&bars->full[i], 4);       // the four transform warps
      mbar_init(&bars->empty[i], 128);    // every thread of the consumer warpgroup
    }
    for (int i = 0; i < 2; ++i) mbar_init(&bars->x_empty[i], 128);
    fence_barrier_init();
  }
  // x ring and W1 panels: the MMAs read 64 columns (and 64 W1 rows per panel); the chunks past Cin
  // and the rows past Chid are never written below, so they are zeroed once here
  for (int i = threadIdx.x; i < (2 * kXbPanel + kNP * kXbWPanel) / 16; i += kXbThreads)
    *reinterpret_cast<uint4*>(smem + p.off_x + 16 * i) = make_uint4(0u, 0u, 0u, 0u);
  __syncthreads();
  // W1 [Chid][Cin] as the dgrad's MN-major B: row k (hidden channel) of panel k / 64, Cin along
  // the 128-byte row
  {
    const int cpr = p.Cin / 8;
    for (int i = threadIdx.x; i < p.Chid * cpr; i += kXbThreads) {
      const int k = i / cpr, c = i % cpr;
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(p.W1 + (size_t)k * p.Cin + 8 * c));
      *reinterpret_cast<uint4*>(smem + p.off_w + (k >> 6) * kXbWPanel + (k & 63) * 128 +
                                ((c ^ (k & 7)) << 4)) = v;
    }
  }
  fence_proxy_async_smem();   // W1 and the zeros are read by wgmma (async proxy)
  __syncthreads();

  if (warp == 0) {
    // ================================ TMA producer ================================
    if (lane == 0) {
      tma_prefetch_desc(&tmDz);
      tma_prefetch_desc(&tmH);
      int stage = 0, phase = 0;
      for (int sl = blockIdx.x; sl < p.slabs; sl += gridDim.x) {
        const int p0 = sl * p.slab_rows, p1 = min(p0 + p.slab_rows, p.M);
        for (int u0 = p0; u0 < p1; u0 += kXbRows) {
          for (int pn = 0; pn < p.panels; ++pn) {
            xb_wait(&bars->empty[stage], phase ^ 1);
            uint8_t* sA = smem + (size_t)stage * kXbStage;
            mbar_arrive_expect_tx(&bars->tma_full[stage], kXbStage);
            tma_load_2d(&tmDz, &bars->tma_full[stage], sA, pn * 64, u0);
            tma_load_2d(&tmH, &bars->tma_full[stage], sA + kXbPanel, pn * 64, u0);
            if (++stage == S) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else if (warp >= 4 && warp < 8) {
    // ============================ consumer warpgroup ============================
    const int w = warp - 4;
    constexpr int NJ = kBN / 8;           // 8-column groups of an accumulator fragment
    float accW[kNP][kBN / 2];
#pragma unroll
    for (int q = 0; q < kNP; ++q)
#pragma unroll
      for (int i = 0; i < kBN / 2; ++i) accW[q][i] = 0.f;
    float accD[2][kBN / 2];
    int stage = 0, phase = 0, it = 0;
    for (int sl = blockIdx.x; sl < p.slabs; sl += gridDim.x) {
     const int p0 = sl * p.slab_rows, p1 = min(p0 + p.slab_rows, p.M);
     for (int u0 = p0; u0 < p1; u0 += kXbRows, ++it) {
      const int xb = it & 1;
      const uint32_t sX = s_x + xb * kXbPanel;
      // residual rows of this thread's dx fragments: requested now, used after the main loop
      uint32_t rv[2][2][NJ];
#pragma unroll
      for (int hf = 0; hf < 2; ++hf)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = u0 + 64 * hf + 16 * w + (lane >> 2) + 8 * h;
#pragma unroll
          for (int j = 0; j < NJ; ++j) {
            const int col = 8 * j + 2 * (lane & 3);
            rv[hf][h][j] = 0u;
            if (p.residual && row < p1 && col < p.Cin)
              rv[hf][h][j] = __ldg(reinterpret_cast<const uint32_t*>(p.residual + (size_t)row * p.Cin + col));
          }
        }
#pragma unroll
      for (int hf = 0; hf < 2; ++hf)
#pragma unroll
        for (int i = 0; i < kBN / 2; ++i) accD[hf][i] = 0.f;
      int prev = 0;
#pragma unroll
      for (int pn = 0; pn < kNP; ++pn) {
        xb_wait(&bars->full[stage], phase);
        const uint32_t sA = s_stage + stage * kXbStage;
        const uint32_t sW = s_w + pn * kXbWPanel;
        reg_fence(accD);
        reg_fence(accW);
        wgmma_fence();
        // dgrad: dh1 panel as the K-major k-block of both 64-row halves, the k order of the
        // two-GEMM dgrad (k-block by k-block, four k16 steps each)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const uint64_t bd = gmma_smem_desc(sW + kk * 2048, kXbWPanel, 1024);
          xb_mma<0, 1, kBN>(accD[0], gmma_smem_desc(sA + kk * 32, 16, 1024), bd);
          xb_mma<0, 1, kBN>(accD[1], gmma_smem_desc(sA + 64 * 128 + kk * 32, 16, 1024), bd);
        }
        // wgrad: the same bytes as the MN-major [64 ch x 128 px] A block, x as MN-major B
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)
          xb_mma<1, 1, kBN>(accW[pn], gmma_smem_desc(sA + kk * 2048, kXbPanel, 1024),
                            gmma_smem_desc(sX + kk * 2048, kXbPanel, 1024));
        wgmma_commit();
        if (pn > 0) {          // the previous panel's wgmmas retired: its stage is free
          wgmma_wait<1>();
          mbar_arrive(&bars->empty[prev]);
        }
        prev = stage;
        if (++stage == S) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      reg_fence(accD);
      reg_fence(accW);
      mbar_arrive(&bars->empty[prev]);
      mbar_arrive(&bars->x_empty[xb]);
      // dx = acc (+ residual), rounded to bf16; rows past the slab (the next slab's, or past M)
      // are not stored
#pragma unroll
      for (int hf = 0; hf < 2; ++hf)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = u0 + 64 * hf + 16 * w + (lane >> 2) + 8 * h;
#pragma unroll
          for (int j = 0; j < NJ; ++j) {
            const int col = 8 * j + 2 * (lane & 3);
            float v0 = accD[hf][4 * j + 2 * h], v1 = accD[hf][4 * j + 2 * h + 1];
            v0 += bf16lo(rv[hf][h][j]);
            v1 += bf16hi(rv[hf][h][j]);
            if (row < p1 && col < p.Cin)
              *reinterpret_cast<uint32_t*>(p.dx + (size_t)row * p.Cin + col) = pack_bf16(v0, v1);
          }
        }
     }
     // the slab's dW1 partial: plain stores (rows past Chid / columns past Cin are padding), then
     // the next slab starts from zero
     float* part = p.part + (size_t)sl * p.Chid * p.Cin;
#pragma unroll
     for (int pn = 0; pn < kNP; ++pn)
#pragma unroll
       for (int h = 0; h < 2; ++h) {
         const int row = 64 * pn + 16 * w + (lane >> 2) + 8 * h;
#pragma unroll
         for (int j = 0; j < NJ; ++j) {
           const int col = 8 * j + 2 * (lane & 3);
           if (row < p.Chid && col < p.Cin)
             __stcg(reinterpret_cast<float2*>(part + (size_t)row * p.Cin + col),
                    make_float2(accW[pn][4 * j + 2 * h], accW[pn][4 * j + 2 * h + 1]));
         }
       }
#pragma unroll
     for (int q = 0; q < kNP; ++q)
#pragma unroll
       for (int i = 0; i < kBN / 2; ++i) accW[q][i] = 0.f;
    }
  } else if (warp >= 8) {
    // =================== transform warps: dh1 in place, x rows by cp.async ===================
    const int tw = warp - 8;              // rows 32 tw .. 32 tw + 31 of every panel
    const int lc = lane & 7;              // the 16-byte chunk (8 channels) this lane owns
    const uint32_t swz = (uint32_t)(lc << 4);
    int stage = 0, phase = 0, it = 0;
    for (int sl = blockIdx.x; sl < p.slabs; sl += gridDim.x) {
     const int p0 = sl * p.slab_rows, p1 = min(p0 + p.slab_rows, p.M);
     for (int u0 = p0; u0 < p1; u0 += kXbRows, ++it) {
      // rows past the slab end (the next slab's, or past M) are zero in dh1 and x: they add
      // nothing to this slab's dW1, as the rows past a split-K slab add nothing to its partial
      const int rlimit = min(kXbRows, p1 - u0);
      const int xb = it & 1;
      // x rows [128 px x Cin] of the unit
      xb_wait(&bars->x_empty[xb], ((it >> 1) & 1) ^ 1);
      {
        const int r = 32 * tw + lane;
        const bool ok = r < rlimit;
        const __nv_bfloat16* src = ok ? p.x + (size_t)(u0 + r) * p.Cin : p.x;
        const uint32_t dst = s_x + xb * kXbPanel + r * 128;
        for (int c = 0; c < p.Cin / 8; ++c)
          cp_async_zfill16(dst + (uint32_t)((c ^ (r & 7)) << 4), ok ? src + 8 * c : src,
                           ok ? 16 : 0);
        cp_async_commit();
      }
      for (int pn = 0; pn < p.panels; ++pn) {
        const int c0 = pn * 64 + lc * 8;
        const bool cok = c0 < p.Chid;
        float2 sc[4], s2[4], sh[4];
        {
          float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, b0 = a0, b1 = a0, t0 = a0, t1 = a0;
          if (cok) {
            a0 = __ldg(reinterpret_cast<const float4*>(p.ca + c0));
            a1 = __ldg(reinterpret_cast<const float4*>(p.ca + c0 + 4));
            t0 = __ldg(reinterpret_cast<const float4*>(p.cb + c0));
            t1 = __ldg(reinterpret_cast<const float4*>(p.cb + c0 + 4));
            b0 = __ldg(reinterpret_cast<const float4*>(p.cc + c0));
            b1 = __ldg(reinterpret_cast<const float4*>(p.cc + c0 + 4));
          }
          sc[0] = make_float2(a0.x, a0.y); sc[1] = make_float2(a0.z, a0.w);
          sc[2] = make_float2(a1.x, a1.y); sc[3] = make_float2(a1.z, a1.w);
          s2[0] = make_float2(t0.x, t0.y); s2[1] = make_float2(t0.z, t0.w);
          s2[2] = make_float2(t1.x, t1.y); s2[3] = make_float2(t1.z, t1.w);
          sh[0] = make_float2(b0.x, b0.y); sh[1] = make_float2(b0.z, b0.w);
          sh[2] = make_float2(b1.x, b1.y); sh[3] = make_float2(b1.z, b1.w);
        }
        xb_wait(&bars->tma_full[stage], phase);
        const uint32_t sA = s_stage + stage * kXbStage;
        uint4 v[8], u[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int r = 32 * tw + (lane >> 3) + 4 * j;
          const uint32_t off = (uint32_t)(r * 128) + (swz ^ (uint32_t)((r & 7) << 4));
          v[j] = lds128(sA + off);
          u[j] = lds128(sA + kXbPanel + off);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int r = 32 * tw + (lane >> 3) + 4 * j;
          const uint32_t off = (uint32_t)(r * 128) + (swz ^ (uint32_t)((r & 7) << 4));
          const uint32_t dv[4] = {v[j].x, v[j].y, v[j].z, v[j].w};
          const uint32_t hv[4] = {u[j].x, u[j].y, u[j].z, u[j].w};
          uint32_t o[4];
          // the GEMM loaders' two-source transform: ca * dz1 + (cb * h1 + cc), RN to bf16
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 t = ffma2(s2[e], make_float2(bf16lo(hv[e]), bf16hi(hv[e])), sh[e]);
            const float2 d = ffma2(sc[e], make_float2(bf16lo(dv[e]), bf16hi(dv[e])), t);
            o[e] = pack_bf16(d.x, d.y);
          }
          // rows past M and channels past Chid stay zero (the TMA's fill)
          const bool ok = cok && r < rlimit;
          sts128(sA + off,
                 make_uint4(ok ? o[0] : 0u, ok ? o[1] : 0u, ok ? o[2] : 0u, ok ? o[3] : 0u));
        }
        if (pn == 0) cp_async_wait<0>();   // x rows landed
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars->full[stage]);
        if (++stage == S) { stage = 0; phase ^= 1; }
      }
     }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
using XbLaunchFn = void (*)(int, int, cudaStream_t, const CUtensorMap&, const CUtensorMap&, const XbDev&);
template <int BN, int NP>
static void xb_launch(int grid, int smem, cudaStream_t st, const CUtensorMap& a, const CUtensorMap& b,
                      const XbDev& p) {
  expand_bwd_kernel<BN, NP><<<grid, kXbThreads, smem, st>>>(a, b, p);
}
template <int BN, int NP>
static const void* xb_fn() { return (const void*)expand_bwd_kernel<BN, NP>; }

struct XbPlan {
  XbDev p;
  int block_n, grid, smem;
  XbLaunchFn fn;
  const void* kern;
};

static int xb_plan(const yamb_expand_bwd_args* a, int num_sms, XbPlan& pl) {
  if (!a) return set_error(YAMB_EINVAL, "expand_bwd: no arguments");
  if (a->M <= 0 || a->Cin < 8 || a->Cin > 32 || a->Chid < 64 || a->Chid > 64 * kXbMaxPanels ||
      (a->Cin % 8) || (a->Chid % 8))
    return set_error(YAMB_EINVAL,
                     "expand_bwd: shape outside the kernel's caps (M=%d Cin=%d Chid=%d; "
                     "8 <= Cin <= 32, 64 <= Chid <= 192, channels multiples of 8)",
                     a->M, a->Cin, a->Chid);
  const int sms = num_sms > 0 ? num_sms : max_ctas();
  if (sms <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  XbDev& p = pl.p;
  memset(&p, 0, sizeof(p));
  p.M = a->M; p.Cin = a->Cin; p.Chid = a->Chid;
  p.panels = (a->Chid + 63) / 64;
  // the slabs of the split-K wgrad GEMM this kernel replaces (dW1[Chid][Cin] += dh1^T x, both
  // operands MN-major, two-source transform of A), from that GEMM's own plan
  {
    static const float coef = 0.f;
    yamb_gemm g;
    memset(&g, 0, sizeof(g));
    g.M = a->Chid; g.N = a->Cin; g.K = a->M;
    g.a_mn_major = g.b_mn_major = 1;
    g.epi = 2;
    g.a_xform = 2;
    g.a_scale = g.a_shift = g.a_scale2 = &coef;
    g.A = g.A2 = g.B = g.D = (void*)&coef;
    g.lda = g.lda2 = a->Chid; g.ldb = g.ldd = a->Cin;
    yamb_gemm_plan_info wi;
    const int rc = gemm_plan_query(&g, sms, &wi);
    if (rc) return rc;
    p.slabs = wi.ksplit;
    p.slab_rows = wi.kb_per_split * 64;
  }
  pl.block_n = a->Cin <= 16 ? 16 : 32;
  const int fixed = 2 * kXbPanel + p.panels * kXbWPanel + (int)sizeof(XbBars);
  const int budget = 232448;   // 227 KB of dynamic shared memory per block
  int stages = (budget - fixed) / kXbStage;
  if (stages > kXbMaxStages) stages = kXbMaxStages;
  p.num_stages = stages;
  p.off_x = stages * kXbStage;
  p.off_w = p.off_x + 2 * kXbPanel;
  p.off_bars = p.off_w + p.panels * kXbWPanel;
  pl.smem = p.off_bars + (int)sizeof(XbBars);
  pl.grid = p.slabs < sms ? p.slabs : sms;
  const int np = p.panels;
  if (pl.block_n == 16) {
    pl.fn = np == 1 ? &xb_launch<16, 1> : np == 2 ? &xb_launch<16, 2> : &xb_launch<16, 3>;
    pl.kern = np == 1 ? xb_fn<16, 1>() : np == 2 ? xb_fn<16, 2>() : xb_fn<16, 3>();
  } else {
    pl.fn = np == 1 ? &xb_launch<32, 1> : np == 2 ? &xb_launch<32, 2> : &xb_launch<32, 3>;
    pl.kern = np == 1 ? xb_fn<32, 1>() : np == 2 ? xb_fn<32, 2>() : xb_fn<32, 3>();
  }
  return 0;
}

static int xb_map(CUtensorMap* map, const void* ptr, int M, int C) {
  static PFN_encodeTiled encode = get_encode_tiled();
  if (!encode) return set_error(YAMB_ECUDA, "cuTensorMapEncodeTiled entry point not found");
  cuuint64_t dims[2] = {(cuuint64_t)C, (cuuint64_t)M};
  cuuint64_t strides[1] = {(cuuint64_t)C * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)kXbRows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides,
                      box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(YAMB_ECUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return 0;
}

int expand_bwd_plan_query(const yamb_expand_bwd_args* a, int num_sms, yamb_expand_bwd_plan_info* out) {
  if (!out) return set_error(YAMB_EINVAL, "no plan output");
  XbPlan pl;
  const int rc = xb_plan(a, num_sms, pl);
  if (rc) return rc;
  memset(out, 0, sizeof(*out));
  out->block_n = pl.block_n;
  out->panels = pl.p.panels;
  out->slabs = pl.p.slabs;
  out->slab_rows = pl.p.slab_rows;
  out->grid = pl.grid;
  out->num_stages = pl.p.num_stages;
  out->smem_bytes = pl.smem;
  return 0;
}

int expand_bwd_launch(const yamb_expand_bwd_args* a, cudaStream_t stream) {
  if (!a) return set_error(YAMB_EINVAL, "expand_bwd: no arguments");
  const void* ptrs[9] = {a->dz1, a->h1, a->ca, a->cb, a->cc, a->W1, a->x, a->dx, a->dW1};
  for (int i = 0; i < 9; ++i)
    if (!ptrs[i] || (reinterpret_cast<uintptr_t>(ptrs[i]) & 15))
      return set_error(YAMB_EINVAL, "expand_bwd: pointer %d is NULL or not 16-byte aligned", i);
  if (a->residual && (reinterpret_cast<uintptr_t>(a->residual) & 15))
    return set_error(YAMB_EINVAL, "expand_bwd: residual not 16-byte aligned");
  XbPlan pl;
  int rc = xb_plan(a, 0, pl);
  if (rc) return rc;
  XbDev& p = pl.p;
  p.ca = a->ca; p.cb = a->cb; p.cc = a->cc;
  p.W1 = (const __nv_bfloat16*)a->W1;
  p.x = (const __nv_bfloat16*)a->x;
  p.residual = (const __nv_bfloat16*)a->residual;
  p.dx = (__nv_bfloat16*)a->dx;
  CUtensorMap tmDz, tmH;
  if ((rc = xb_map(&tmDz, a->dz1, a->M, a->Chid))) return rc;
  if ((rc = xb_map(&tmH, a->h1, a->M, a->Chid))) return rc;
  if ((rc = smem_optin("expand_bwd launch", pl.kern, pl.smem))) return rc;
  if ((rc = det_alloc((size_t)p.slabs * a->Chid * a->Cin * sizeof(float), stream, &p.part))) return rc;
  pl.fn(pl.grid, pl.smem, stream, tmDz, tmH, p);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    det_free(p.part, stream);
    return set_error(YAMB_ECUDA, "expand_bwd launch: %s", cudaGetErrorString(e));
  }
  return det_reduce_launch(p.part, p.slabs, (long long)a->Chid * a->Cin, a->dW1, stream, true);
}

}  // namespace yamb
