// Pointwise-convolution GEMM for sm_90a: operand loaders -> shared memory -> wgmma -> registers ->
// epilogue.
//
// One persistent CTA (512 threads) per SM, warp-specialised:
//   warp 0      TMA producer for WIDE TRANSFORMED operands only (128-byte box rows)
//   warps 1-3   barrier set-up, then idle
//   warps 4-11  two consumer warpgroups that alternate tiles: each runs the wgmma main loop of its
//               tile (128 x block_n, two m64 halves, fp32 accumulators in registers) and then its
//               epilogue, while the other warpgroup runs the next tile's main loop.  A turn barrier
//               hands the main loop over, so the k-blocks are consumed in ring order.  Every WARP's
//               epilogue is independent: registers -> fused math -> warp-private swizzled smem ->
//               its own TMA stores (two boxes of 64 x 16) -> per-column BatchNorm statistics read
//               back from the staged tile.  No CTA-wide barrier in the steady state.
//   warps 12-15 (and 8-11 when the epilogue is light) operand loaders: one warp per pipeline stage;
//               plain operands by cp.async into the swizzled layout, narrow transformed operands
//               through registers, wide transformed operands rewritten in place after the TMA
//               landed them (BN-apply + activation, or the two-source BN-backward affine)
// (TMA tile loads cost several cycles per box row whatever its width: with the 32-96-byte rows of
// the narrow operands the TMA unit would bound the GEMM, so those go through cp.async.)
//
// Replaces, behind yamb_pointwise_gemm (include/yamb200.h), the nn.Conv2d(kernel_size=1) forward /
// dgrad / wgrad library calls of the reference block (models/mobilenet_base.py:391-395, :413,
// :253-257, :284-285) together with the BatchNorm statistics passes (:203, :417).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <string.h>

#include "bn_finalize.cuh"
#include "host_util.h"
#include "prims.cuh"

namespace yamb {
// Why the last mbarrier wait of gemm_tc_kernel that gave up did so:
//   bits 40..63 block, 24..39 thread, 0..23 shared-memory address of the barrier.
// Zero while no wait has timed out; readable from a debugger or a GPU core dump after the trap.
__device__ unsigned long long g_gemm_wait_timeout;

// Bounded mbarrier wait without a call in it: the printf of mbar_wait is an out-of-line call, and a
// call inside the window where wgmmas are in flight makes ptxas serialise the whole wgmma sequence
// (C7520).  A pipeline bug still traps after ~4 s instead of hanging the GPU.
__device__ __forceinline__ void gemm_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = global_timer_ns();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (((++spins) & 0x3fff) == 0 && global_timer_ns() - t0 > 4000000000ull) {
      *reinterpret_cast<volatile unsigned long long*>(&g_gemm_wait_timeout) =
          ((unsigned long long)blockIdx.x << 40) | ((unsigned long long)(threadIdx.x & 0xffff) << 24) |
          (smem_u32(bar) & 0xffffffu);
      __threadfence_system();
      __trap();
    }
  }
}


constexpr int kBlockM = 128;
constexpr int kBlockK = 64;          // 64 bf16 = 128 bytes = one SWIZZLE_128B row
constexpr int kPanelBytes64 = 8192;  // 64 rows x 128 B
constexpr int kABytes = 16384;       // 128 x 64 bf16
constexpr int kWarpOutBytes = 4096;  // 32 rows x 64 cols bf16: one warp's staging sub-tile
constexpr int kEpiWarps = 8;
constexpr int kMaxStages = 8;
constexpr int kMaxBlockN = 64;    // 2 x 32 fp32 accumulators per thread of a consumer warpgroup

struct GemmDev {
  int M, N, K;
  int block_n, m_blocks, n_blocks, num_k_blocks, ksplit, kb_per_split, num_work;
  int a_mn, b_mn;
  int num_stages;
  int a_bytes;      // bytes of the A region of one stage (8 KB when an MN-major A has <= 64 rows)
  int b_bytes;      // bytes of the B region of one stage
  int a2_off;       // offset of A2 region inside a stage (0 = none)
  int b2_off;
  int stage_bytes;
  int a_xform, a_act, b_xform, b_act;
  const float *a_scale, *a_shift, *a_scale2;
  const float *b_scale, *b_shift, *b_scale2;
  int epi;
  int has_residual;
  void* D;
  long long ldd;
  const __nv_bfloat16* side;  // residual (epi 0) or H (epi 1), row-major [M][lds]
  long long lds;
  int out_bufs;               // staging buffers per epilogue warp (1 or 2)
  const float *a_gate, *b_gate;  // optional per-(sample, channel) gates [n][C] (SE)
  long long gate_rps;            // pixels per sample
  int wg2x;                   // 1: warps 8-11 transform (light epilogue), 0: they are epilogue WG 1
  // operand tensors in global memory ([pixels|rows][channels], bf16) for the cp.async loaders
  const __nv_bfloat16 *gA, *gA2, *gB, *gB2;
  long long lda, lda2, ldb, ldb2;
  int a_tma, b_tma;           // wide transformed operand: TMA load + in-place smem transform
  int lgroup;                 // loader warps that share one stage (1, 2 or 4)
  float* part;                // epi 2: [num_work][128][64] fp32 split-K partial tiles
  yamb_bn_fwd bnf;
  int has_bnf;
  const float *h_scale, *h_shift;
  int h_act;
  yamb_bn_bwd bnb;
  int has_bnb;
  // smem offsets (bytes from the 1024-aligned base)
  int off_out, off_hside, off_coef, off_stats, off_bars;
};

struct Bars {
  uint64_t full[kMaxStages];
  uint64_t xdone[kMaxStages];
  uint64_t empty[kMaxStages];
  uint64_t turn[2];   // main-loop hand-over between the two consumer warpgroups
};

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Register-staged load + transform of one operand panel by ONE warp: every lane owns the same
// 8-channel column (lc = lane & 7) for the whole panel, so its BatchNorm / affine coefficients sit
// in registers; 8 rows (16-byte vectors) per lane are in flight from global memory at a time, are
// transformed in registers and stored straight into the SWIZZLE_128B layout (no shared-memory
// round trip, no cross-warp synchronisation).
//   mode 1: v = act(s[c]*v + b[c]) [* gate]      mode 2: v = s[c]*v + s2[c]*v2 + b[c]
// Vectors outside the tensor (row >= rlimit or channel >= C) are stored as zero.
template <int MODE, bool SMEM>
__device__ __forceinline__ void gxform_panel(uint32_t panel, uint32_t panel2, const __nv_bfloat16* g1, long long ld1,
                                             const __nv_bfloat16* g2, long long ld2, int rbeg, int rows,
                                             int rlimit, int ln, int cs, const ActParam& ap,
                                             uint32_t tab_s, uint32_t tab_b, uint32_t tab_s2,
                                             int col0, int C, const float* gate, unsigned pixbase,
                                             unsigned rps) {
  // rows in flight per lane (16 B each, x2 sources in mode 2).  From global memory every batch
  // exposes one DRAM latency to this warp: keep the batch as large as the registers allow.
  constexpr int NB = (MODE == 2 && SMEM) ? 4 : 8;
  // 2^cs lanes per row (8 for 64-channel panels; 4 / 2 for narrow operands so that no lane idles)
  const int lc = ln & ((1 << cs) - 1);
  const int RS = 32 >> cs;                // rows covered by one warp-wide access
  const int c0 = col0 + lc * 8;
  const bool cok = c0 < C;
  float2 sc[4], sh[4], s2[4];
  {
    float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, b0 = a0, b1 = a0, t0 = a0, t1 = a0;
    if (cok) {
      a0 = lds128f(tab_s + c0 * 4); a1 = lds128f(tab_s + c0 * 4 + 16);
      b0 = lds128f(tab_b + c0 * 4); b1 = lds128f(tab_b + c0 * 4 + 16);
      if (MODE == 2) { t0 = lds128f(tab_s2 + c0 * 4); t1 = lds128f(tab_s2 + c0 * 4 + 16); }
    }
    sc[0] = make_float2(a0.x, a0.y); sc[1] = make_float2(a0.z, a0.w);
    sc[2] = make_float2(a1.x, a1.y); sc[3] = make_float2(a1.z, a1.w);
    sh[0] = make_float2(b0.x, b0.y); sh[1] = make_float2(b0.z, b0.w);
    sh[2] = make_float2(b1.x, b1.y); sh[3] = make_float2(b1.z, b1.w);
    s2[0] = make_float2(t0.x, t0.y); s2[1] = make_float2(t0.z, t0.w);
    s2[2] = make_float2(t1.x, t1.y); s2[3] = make_float2(t1.z, t1.w);
  }
  const uint32_t lo2 = pack_bf16(ap.lo, ap.lo), hi2 = pack_bf16(ap.hi, ap.hi);
  const __nv_bfloat16* p1 = g1 + c0;
  const __nv_bfloat16* p2 = g2 + c0;
  // Straight-line batches (no per-chunk branches: the NB chunk bodies interleave, one warp has
  // NB independent dependency chains in flight; with a branch per chunk a loader warp ran at
  // ~0.1 IPC and the loaders bounded the GEMM).  `lean`: clamp-type activation, no SE gate.
  const bool lean = ap.kind == 0 && gate == nullptr;
  const uint32_t swz = (uint32_t)(lc << 4);
  const float inv_rps = pixbase < (1u << 24) - 1024u ? 1.0f / (float)rps : 0.f;   // 0: divide
#pragma unroll 1
  for (int rb = rbeg + (ln >> cs); rb < rows; rb += RS * NB) {
    uint4 v[NB], w[MODE == 2 ? NB : 1];
#pragma unroll
    for (int j = 0; j < NB; ++j) {
      const int r = rb + RS * j;
      const bool ok = cok && r < rlimit;
      if (SMEM) {   // the TMA producer put the raw tile(s) there: rewrite in place
        const uint32_t off = (uint32_t)(r * 128) + (swz ^ (uint32_t)((r & 7) << 4));
        const bool in = r < rows;   // (always a valid shared address; value unused otherwise)
        v[j] = in ? lds128(panel + off) : make_uint4(0u, 0u, 0u, 0u);
        if (MODE == 2) w[j] = in ? lds128(panel2 + off) : make_uint4(0u, 0u, 0u, 0u);
      } else {
        v[j] = make_uint4(0u, 0u, 0u, 0u);
        if (MODE == 2) w[j] = make_uint4(0u, 0u, 0u, 0u);
        if (ok) {
          v[j] = __ldg(reinterpret_cast<const uint4*>(p1 + (long long)r * ld1));
          if (MODE == 2) w[j] = __ldg(reinterpret_cast<const uint4*>(p2 + (long long)r * ld2));
        }
      }
    }
    uint32_t o[NB][4];
    if (MODE == 2) {
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        const uint32_t xv[4] = {v[j].x, v[j].y, v[j].z, v[j].w};
        const uint32_t yv[4] = {w[j].x, w[j].y, w[j].z, w[j].w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 t1 = ffma2(s2[e], make_float2(bf16lo(yv[e]), bf16hi(yv[e])), sh[e]);
          const float2 d = ffma2(sc[e], make_float2(bf16lo(xv[e]), bf16hi(xv[e])), t1);
          o[j][e] = pack_bf16(d.x, d.y);
        }
      }
    } else if (lean) {
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        const uint32_t xv[4] = {v[j].x, v[j].y, v[j].z, v[j].w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 d = ffma2(sc[e], make_float2(bf16lo(xv[e]), bf16hi(xv[e])), sh[e]);
          o[j][e] = clamp_bf16x2(pack_bf16(d.x, d.y), lo2, hi2);
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < NB; ++j) {   // swish / h-swish / SE gate
        const int r = rb + RS * j;
        const uint32_t xv[4] = {v[j].x, v[j].y, v[j].z, v[j].w};
        float x[8];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 d = ffma2(sc[e], make_float2(bf16lo(xv[e]), bf16hi(xv[e])), sh[e]);
          x[2 * e] = d.x; x[2 * e + 1] = d.y;
        }
        act_vec<8>(x, ap);
        if (gate != nullptr && cok && r < rlimit) {
          // SE: the gate multiplies the bf16-rounded activation (oracle rounding points)
          // sample index = pixel / pixels-per-sample without an integer division: float reciprocal
          // (pixel indices < 2^24 are exact in fp32) and a one-step correction either way
          const unsigned pix = pixbase + (unsigned)r;
          unsigned smp;
          if (inv_rps != 0.f) {
            smp = (unsigned)__fmul_rz((float)pix, inv_rps);
            if (smp * rps > pix) --smp;
            else if ((smp + 1u) * rps <= pix) ++smp;
          } else {
            smp = pix / rps;
          }
          const float* gr = gate + (size_t)smp * C + c0;
          const float4 q0 = __ldg(reinterpret_cast<const float4*>(gr));
          const float4 q1 = __ldg(reinterpret_cast<const float4*>(gr + 4));
          const float gq[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
          for (int e = 0; e < 8; ++e) x[e] = round_bf16(x[e]) * gq[e];
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) o[j][e] = pack_bf16(x[2 * e], x[2 * e + 1]);
      }
    }
#pragma unroll
    for (int j = 0; j < NB; ++j) {
      const int r = rb + RS * j;
      const bool ok = cok && r < rlimit;
      if (r < rows)
        sts128(panel + (uint32_t)(r * 128) + (swz ^ (uint32_t)((r & 7) << 4)),
               make_uint4(ok ? o[j][0] : 0u, ok ? o[j][1] : 0u, ok ? o[j][2] : 0u, ok ? o[j][3] : 0u));
    }
  }
}

// One k16 step of a 64-row half: d[0 .. BN/2) (+)= A * B with the wgmma of width BN.
template <int TA, int TB, int BN>
__device__ __forceinline__ void mma_bn(float (&d)[32], uint64_t ad, uint64_t bd) {
  if constexpr (BN == 64) wgmma_m64n64<TA, TB>(d, ad, bd, 1u);
  else if constexpr (BN == 32) wgmma_m64n32<TA, TB>(reinterpret_cast<float(&)[16]>(d), ad, bd, 1u);
  else wgmma_m64n16<TA, TB>(reinterpret_cast<float(&)[8]>(d), ad, bd, 1u);
}

// kBN (block_n = wgmma width), kAmn / kBmn (operand majors) are compile-time so that the consumer's
// wgmma sequence is straight-line code: a runtime choice of instruction, a branch around the upper
// half or a runtime k16 count puts the wgmmas in divergent paths, and ptxas then serialises every
// one of them (C7520).  gemm_launch instantiates only the combinations the layers produce.
template <bool kXform, int kEpi, int kBN, int kAmn, int kBmn>
__global__ void __launch_bounds__(512, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
               const __grid_constant__ CUtensorMap tmD, const __grid_constant__ GemmDev p) {
  // 1024-byte alignment (SWIZZLE_128B atoms) comes from the declaration, not from pointer
  // arithmetic, so the compiler keeps every access in the shared address space (LDS/STS, not
  // generic LD/ST).
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw;
  Bars* bars = reinterpret_cast<Bars*>(smem + p.off_bars);
  stat_t* s_stats = reinterpret_cast<stat_t*>(smem + p.off_stats);  // [2][N], double
  float* s_coef = reinterpret_cast<float*>(smem + p.off_coef);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int S = p.num_stages;

  // ---- one-time setup ------------------------------------------------------------------------
  if (warp == 0 && lane == 0) {
    if (kEpi != 2) tma_prefetch_desc(&tmD);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < S; ++i) {
      mbar_init(&bars->full[i], p.lgroup);   // the loader warps that own the stage arrive
      mbar_init(&bars->xdone[i], 1);
      mbar_init(&bars->empty[i], 128);       // every thread of the consuming warpgroup arrives
    }
    for (int i = 0; i < 2; ++i) mbar_init(&bars->turn[i], 1);
    fence_barrier_init();
  }
  // zero the per-CTA statistics accumulators
  if (p.has_bnf || p.has_bnb) {
    for (int i = threadIdx.x; i < 2 * p.N; i += blockDim.x) s_stats[i] = 0.0;
  }
  // The MMA reads all 64 columns (4 k16 steps) of every k-block.  A K-major operand of K <= 32
  // is loaded into 2 or 4 of the 8 16-byte chunks of each row only (panel_of: cshift); nothing
  // else writes the other chunks during the launch, so they are zeroed once here.
  if (p.K <= 32 && (!kAmn || !kBmn)) {
    for (int i = threadIdx.x; i < S * p.stage_bytes / 16; i += blockDim.x)
      sts128(smem_u32(smem) + 16u * (uint32_t)i, make_uint4(0u, 0u, 0u, 0u));
    fence_proxy_async_smem();   // the zeros are read by wgmma (async proxy)
  }
  __syncthreads();

  const bool use_x = kXform && (p.a_xform != 0 || p.b_xform != 0);

  // 512-thread variant: every thread starts with 128 registers; the control warpgroup hands its
  // surplus to the consumer and loader warps (56*4 + 152*12 warps x 32 lanes = 64 Ki regs).
  if (warp < 4) {
   asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
   if (warp == 0) {
    // ============ TMA producer: wide transformed operands only (128-byte box rows) ============
    if (lane == 0 && (p.a_tma || p.b_tma)) {
      tma_prefetch_desc(&tmA);
      tma_prefetch_desc(&tmB);
      int stage = 0, phase = 0;
      for (int w = blockIdx.x; w < p.num_work; w += gridDim.x) {
        const int mn = w / p.ksplit, slab = w % p.ksplit;
        const int m_blk = mn / p.n_blocks, n_blk = mn % p.n_blocks;
        const int kb0 = slab * p.kb_per_split;
        const int kb1 = min(kb0 + p.kb_per_split, p.num_k_blocks);
        for (int kb = kb0; kb < kb1; ++kb) {
          gemm_wait(&bars->empty[stage], phase ^ 1);
          uint8_t* sA = smem + (size_t)stage * p.stage_bytes;
          uint8_t* sB = sA + p.a_bytes;
          uint32_t tx = 0;
          const int a_panels = kAmn ? 2 : 1;
          int a_issue[2] = {0, 0};
          const int b_panels = (kBN + 63) / 64;
          if (p.a_tma) {
            if (!kAmn) {
              tx += (uint32_t)kABytes;
            } else {
              for (int q = 0; q < 2; ++q)
                if (m_blk * kBlockM + q * 64 < p.M) { a_issue[q] = 1; tx += kPanelBytes64; }
            }
            if (p.a_xform == 2) tx += kAmn ? (a_issue[0] + a_issue[1]) * kPanelBytes64 : (uint32_t)kABytes;
          }
          if (p.b_tma) {
            uint32_t tb = 0;
            if (!kBmn) {
              tb = (uint32_t)kBN * 128u;
            } else {
              for (int q = 0; q < b_panels; ++q)
                if (n_blk * kBN + q * 64 < p.N) tb += kPanelBytes64;
            }
            tx += p.b_xform == 2 ? 2 * tb : tb;
          }
          mbar_arrive_expect_tx(&bars->xdone[stage], tx);
          if (p.a_tma) {
            if (!kAmn) {
              tma_load_2d(&tmA, &bars->xdone[stage], sA, kb * kBlockK, m_blk * kBlockM);
              if (p.a_xform == 2)
                tma_load_2d(&tmA2, &bars->xdone[stage], sA + p.a2_off, kb * kBlockK, m_blk * kBlockM);
            } else {
              for (int q = 0; q < a_panels; ++q)
                if (a_issue[q]) {
                  tma_load_2d(&tmA, &bars->xdone[stage], sA + q * kPanelBytes64,
                              m_blk * kBlockM + q * 64, kb * kBlockK);
                  if (p.a_xform == 2)
                    tma_load_2d(&tmA2, &bars->xdone[stage], sA + p.a2_off + q * kPanelBytes64,
                                m_blk * kBlockM + q * 64, kb * kBlockK);
                }
            }
          }
          if (p.b_tma) {
            if (!kBmn) {
              tma_load_2d(&tmB, &bars->xdone[stage], sB, kb * kBlockK, n_blk * kBN);
              if (p.b_xform == 2)
                tma_load_2d(&tmB2, &bars->xdone[stage], sA + p.b2_off, kb * kBlockK,
                            n_blk * kBN);
            } else {
              for (int q = 0; q < b_panels; ++q)
                if (n_blk * kBN + q * 64 < p.N) {
                  tma_load_2d(&tmB, &bars->xdone[stage], sB + q * kPanelBytes64,
                              n_blk * kBN + q * 64, kb * kBlockK);
                  if (p.b_xform == 2)
                    tma_load_2d(&tmB2, &bars->xdone[stage], sA + p.b2_off + q * kPanelBytes64,
                                n_blk * kBN + q * 64, kb * kBlockK);
                }
            }
          }
          if (++stage == S) { stage = 0; phase ^= 1; }
        }
      }
    }
   }
  } else if (warp < 8 || (warp < 12 && !(kXform && p.wg2x))) {
    // ============================ consumers: wgmma main loop + epilogue ============================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 152;");
    const int ew = warp - 4;           // 0..7
    const int wg = ew >> 2;            // consumer warpgroup
    const int q = warp & 3;            // warp of the warpgroup: rows 16q..16q+15 of each 64-row half
    const int ctid = threadIdx.x & 127;
    uint8_t* s_out = smem + p.off_out + (size_t)ew * p.out_bufs * kWarpOutBytes;
    uint8_t* s_h = smem + p.off_hside + (size_t)ew * kWarpOutBytes;  // side rows (residual / H)
    // per-column coefficient tables for epi 1:  [h_scale | h_shift | mean | invstd] x N
    const float* cz_s = s_coef;
    const float* cz_t = s_coef + p.N;
    const float* cz_m = s_coef + 2 * p.N;
    const float* cz_r = s_coef + 3 * p.N;
    if (kEpi == 1) {
      float* wr = s_coef;
      const int n_epi_thr = (kXform && p.wg2x) ? 128 : 256;
      for (int i = threadIdx.x - 128; i < p.N; i += n_epi_thr) {
        wr[i] = p.h_scale[i];
        wr[p.N + i] = p.h_shift[i];
        wr[2 * p.N + i] = p.bnb.mean[i];
        wr[3 * p.N + i] = p.bnb.invstd[i];
      }
      named_bar_sync(1, n_epi_thr);
    }
    const int n_epi_wg = (kXform && p.wg2x) ? 1 : 2;
    uint32_t sub_count = 0;   // running sub-tile counter of this warp -> staging buffer parity
    const bool side_in = (kEpi == 1) || p.has_residual;
    const ActParam hap = make_act(kEpi == 1 ? p.h_act : ACT_NONE);
    // A warp stages 32 rows of a tile: staged row r <-> tile row 64 * (r >> 4) + 16 q + (r & 15)
    // (the rows of its wgmma accumulator fragments in the two 64-row halves).
    const int lane_trow = (lane >> 4) * 64 + q * 16 + (lane & 15);
    // Column statistics: with a single n-block every lane owns the same 2 columns of sub-tile j in
    // every tile, so the sums live in registers for the whole kernel (shared-memory float atomics
    // are CAS loops and serialise the 8 epilogue warps); flushed once at the end.
    const bool reg_stats = (p.has_bnf || p.has_bnb) && p.n_blocks == 1;
    float racc[kMaxBlockN / 64][4];
#pragma unroll
    for (int j = 0; j < kMaxBlockN / 64; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) racc[j][e] = 0.f;
    // Side operand (residual / H) rows come straight from global memory (lane r loads staged row r:
    // 8 x 16 B per 64-column sub-tile).  They are requested ONE SUB-TILE AHEAD, into the registers
    // the previous sub-tile has just finished with, so their latency hides behind the math.
    uint4 sv[8];
    auto load_side = [&](int w2, int sub2) {
      const int mn2 = w2 / p.ksplit;
      const int m2 = mn2 / p.n_blocks, n2 = mn2 % p.n_blocks;
      const int grow2 = m2 * kBlockM + lane_trow;
      const int col2 = n2 * kBN + sub2 * 64;
      const __nv_bfloat16* srow = p.side + (size_t)grow2 * p.lds + col2;
#pragma unroll
      for (int ch = 0; ch < 8; ++ch) {
        sv[ch] = make_uint4(0u, 0u, 0u, 0u);
        if (grow2 < p.M && col2 + ch * 8 < p.N)
          sv[ch] = __ldg(reinterpret_cast<const uint4*>(srow + ch * 8));
      }
    };
    const int w_step = (n_epi_wg == 2 ? 2 : 1) * (int)gridDim.x;
    if (side_in) {
      const int w0 = blockIdx.x + ((n_epi_wg == 2 && wg == 1) ? (int)gridDim.x : 0);
      if (w0 < p.num_work) load_side(w0, 0);
    }
    float acc[2][32];
    int stage = 0, phase = 0, it = 0;
    uint32_t turn_par = 0;
    for (int w = blockIdx.x; w < p.num_work; w += gridDim.x, ++it) {
      const int mn = w / p.ksplit, slab = w % p.ksplit;
      const int kb0 = slab * p.kb_per_split;
      const int kb1 = min(kb0 + p.kb_per_split, p.num_k_blocks);
      if (n_epi_wg == 2 && (it & 1) != wg) {   // the other warpgroup owns this tile: skip its stages
        stage += kb1 - kb0;
        while (stage >= S) { stage -= S; phase ^= 1; }
        continue;
      }
      const int m_blk = mn / p.n_blocks, n_blk = mn % p.n_blocks;
      // ---- main loop ----
      if (n_epi_wg == 2 && it > 0) {
        gemm_wait(&bars->turn[wg], turn_par);
        turn_par ^= 1;
      }
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[h][i] = 0.f;
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        gemm_wait(&bars->full[stage], phase);
        const uint32_t sA = smem_u32(smem + (size_t)stage * p.stage_bytes);
        const uint32_t sB = sA + p.a_bytes;
        reg_fence(acc[0]);
        reg_fence(acc[1]);
        wgmma_fence();
        // Both 64-row halves and all four k16 steps, unconditionally.  The loaders store zeros
        // past K (the k16 steps past K add exact zeros); rows past M (a missing upper half, or the
        // second panel of an MN-major A of <= 64 channels, which aliases the B region) only feed
        // outputs that are never stored, and the epilogue stages them as zero for the statistics.
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const uint64_t bd = kBmn ? gmma_smem_desc(sB + kk * 2048, kPanelBytes64, 1024)
                                   : gmma_smem_desc(sB + kk * 32, 16, 1024);
          mma_bn<kAmn, kBmn, kBN>(acc[0], kAmn ? gmma_smem_desc(sA + kk * 2048, kPanelBytes64, 1024)
                                               : gmma_smem_desc(sA + kk * 32, 16, 1024), bd);
          mma_bn<kAmn, kBmn, kBN>(acc[1],
                                  kAmn ? gmma_smem_desc(sA + kPanelBytes64 + kk * 2048, kPanelBytes64, 1024)
                                       : gmma_smem_desc(sA + 64 * 128 + kk * 32, 16, 1024), bd);
        }
        wgmma_commit();
        if (prev >= 0) {            // the previous k-block's MMAs retired: its stage is free
          wgmma_wait<1>();
          mbar_arrive(&bars->empty[prev]);
        }
        prev = stage;
        if (++stage == S) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      reg_fence(acc[0]);
      reg_fence(acc[1]);
      if (prev >= 0) mbar_arrive(&bars->empty[prev]);
      if (n_epi_wg == 2 && ctid == 0) mbar_arrive(&bars->turn[wg ^ 1]);   // next tile's main loop
      // ---- epilogue ----
      // sub-tiles of 64 columns; skip the ones that lie entirely beyond N (last n-block)
      const int n_sub = min((kBN + 63) / 64, (p.N - n_blk * kBN + 63) / 64);
#pragma unroll
      for (int sub = 0; sub < kMaxBlockN / 64; ++sub) {
        if (sub >= n_sub) break;
        const int col0 = n_blk * kBN + sub * 64;  // global column of this sub-tile
        if (kEpi == 2) {
          // split-K partial sums: plain stores of the fp32 tile into slab w of the scratch; the
          // reduction kernel that follows adds the slabs into D in slab order (deterministic)
          float* part = p.part + (size_t)w * (kBlockM * kMaxBlockN);
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int r = 64 * h + 16 * q + (lane >> 2) + 8 * e;
#pragma unroll
              for (int jj = 0; jj < 8; ++jj)
                __stcg(reinterpret_cast<float2*>(part + r * kMaxBlockN + sub * 64 + jj * 8 + 2 * (lane & 3)),
                       make_float2(acc[h][4 * (sub * 8 + jj) + 2 * e], acc[h][4 * (sub * 8 + jj) + 2 * e + 1]));
            }
          continue;
        }
        uint8_t* sO = s_out + (p.out_bufs == 2 ? (sub_count & 1) : 0) * kWarpOutBytes;
        // the TMA store that last read this staging buffer must have drained; the previous
        // sub-tile's statistics reads of s_h are behind the __syncwarp that ends it
        if (lane == 0) {
          if (p.out_bufs == 2) tma_store_wait_read<1>();
          else tma_store_wait_read<0>();
        }
        if (side_in) {
#pragma unroll
          for (int ch = 0; ch < 8; ++ch)
            *reinterpret_cast<uint4*>(s_h + lane * 128 + ((ch ^ (lane & 7)) << 4)) = sv[ch];
        }
        __syncwarp();
        // fragments -> bf16 staged tile (row r at r * 128, 16-byte chunks swizzled by r & 7).
        // Rows past M are staged as zero: the statistics below then sum all 32 rows.
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int r = 16 * h + (lane >> 2) + 8 * e;
            const bool rok = m_blk * kBlockM + 64 * h + 16 * q + (lane >> 2) + 8 * e < p.M;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int off = r * 128 + ((jj ^ (r & 7)) << 4) + ((lane & 3) << 2);
              float v0 = acc[h][4 * (sub * 8 + jj) + 2 * e];
              float v1 = acc[h][4 * (sub * 8 + jj) + 2 * e + 1];
              if (kEpi == 1) {
                const uint32_t hh = *reinterpret_cast<const uint32_t*>(s_h + off);
                // columns past N: read the last valid coefficients (the values are never stored)
                const int cb = min(col0 + jj * 8 + 2 * (lane & 3), p.N - 2);
                const float z0 = fmaf(cz_s[cb], bf16lo(hh), cz_t[cb]);
                const float z1 = fmaf(cz_s[cb + 1], bf16hi(hh), cz_t[cb + 1]);
                if (hap.kind == 0) {
                  v0 = (z0 > hap.lo && z0 < hap.hi) ? v0 : 0.f;
                  v1 = (z1 > hap.lo && z1 < hap.hi) ? v1 : 0.f;
                } else {
                  v0 *= act_bwd(z0, p.h_act);
                  v1 *= act_bwd(z1, p.h_act);
                }
              } else if (side_in) {
                const uint32_t rr = *reinterpret_cast<const uint32_t*>(s_h + off);
                v0 += bf16lo(rr);
                v1 += bf16hi(rr);
              }
              *reinterpret_cast<uint32_t*>(sO + off) = rok ? pack_bf16(v0, v1) : 0u;
            }
          }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) {
          tma_store_2d(&tmD, sO, col0, m_blk * kBlockM + q * 16);
          tma_store_2d(&tmD, sO + 2048, col0, m_blk * kBlockM + 64 + q * 16);
          tma_store_commit();
        }
        if (side_in) {
          // request the next sub-tile's side rows now; they land during the statistics pass and
          // the next tile's main loop
          if (sub + 1 < n_sub) load_side(w, sub + 1);
          else if (w + w_step < p.num_work) load_side(w + w_step, 0);
        }
        // ---- per-column statistics of this warp's 32 rows of the bf16-rounded output ----
        if (p.has_bnf || p.has_bnb) {
          const int c = col0 + 2 * lane;  // column pair owned by this lane
          if (c < p.N && (sub * 64 + 2 * lane) < kBN) {
            float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
            const float2 one2 = make_float2(1.f, 1.f), zero2 = make_float2(0.f, 0.f);
            // 4 independent accumulator sets (a 32-deep dependent chain of LDS -> FADD/FFMA would
            // sit on the epilogue's critical path)
            float2 sA = zero2, sB = zero2, sC = zero2, sD = zero2;
            float2 qA = zero2, qB = zero2, qC = zero2, qD = zero2;
            if (p.has_bnf) {
              auto rowf = [&](int r, float2& Sx, float2& Qx) {
                const uint32_t u = *reinterpret_cast<const uint32_t*>(
                    sO + r * 128 + (((lane >> 2) ^ (r & 7)) << 4) + ((lane & 3) << 2));
                const float2 v = make_float2(bf16lo(u), bf16hi(u));
                Sx = ffma2(one2, v, Sx);
                Qx = ffma2(v, v, Qx);
              };
#pragma unroll
              for (int r = 0; r < 32; r += 4) {
                rowf(r, sA, qA);
                rowf(r + 1, sB, qB);
                rowf(r + 2, sC, qC);
                rowf(r + 3, sD, qD);
              }
            } else {
              // sum(dz), sum(dz * xhat) with xhat = h * r - m * r
              const float2 r2 = make_float2(cz_r[c], cz_r[c + 1]);
              const float2 nmr2 = make_float2(-cz_m[c] * r2.x, -cz_m[c + 1] * r2.y);
              auto rowacc = [&](int r, float2& Sx, float2& Qx) {
                const int off = r * 128 + (((lane >> 2) ^ (r & 7)) << 4) + ((lane & 3) << 2);
                const uint32_t u = *reinterpret_cast<const uint32_t*>(sO + off);
                const uint32_t hh = *reinterpret_cast<const uint32_t*>(s_h + off);
                const float2 a = make_float2(bf16lo(u), bf16hi(u));
                const float2 xh = ffma2(make_float2(bf16lo(hh), bf16hi(hh)), r2, nmr2);
                Sx = ffma2(one2, a, Sx);
                Qx = ffma2(a, xh, Qx);
              };
#pragma unroll 2
              for (int r = 0; r < 32; r += 4) {
                rowacc(r, sA, qA);
                rowacc(r + 1, sB, qB);
                rowacc(r + 2, sC, qC);
                rowacc(r + 3, sD, qD);
              }
            }
            s0 = (sA.x + sB.x) + (sC.x + sD.x); s1 = (sA.y + sB.y) + (sC.y + sD.y);
            q0 = (qA.x + qB.x) + (qC.x + qD.x); q1 = (qA.y + qB.y) + (qC.y + qD.y);
            if (reg_stats) {
              racc[sub][0] += s0; racc[sub][1] += s1; racc[sub][2] += q0; racc[sub][3] += q1;
            } else {
              atomicAdd(&s_stats[c], (stat_t)s0);
              atomicAdd(&s_stats[c + 1], (stat_t)s1);
              atomicAdd(&s_stats[p.N + c], (stat_t)q0);
              atomicAdd(&s_stats[p.N + c + 1], (stat_t)q1);
            }
          }
        }
        __syncwarp();  // s_h / sO reads done before the next sub-tile overwrites them
        ++sub_count;
      }
    }
    if (reg_stats) {
#pragma unroll
      for (int j = 0; j < kMaxBlockN / 64; ++j) {
        const int c = j * 64 + 2 * lane;
        if (c < p.N) {
          atomicAdd(&s_stats[c], (stat_t)racc[j][0]);
          atomicAdd(&s_stats[c + 1], (stat_t)racc[j][1]);
          atomicAdd(&s_stats[p.N + c], (stat_t)racc[j][2]);
          atomicAdd(&s_stats[p.N + c + 1], (stat_t)racc[j][3]);
        }
      }
    }
    if (lane == 0 && kEpi != 2) tma_store_wait_all<0>();
  } else {
    // ============================ operand loaders (+ transform) ============================
    // Warps 12-15 (t 0..127) plus, when wg2x, warps 8-11 (t 128..255) bring the operand tiles into
    // shared memory: plain operands with cp.async (16-byte chunks written straight into the
    // SWIZZLE_128B layout the UMMA descriptors expect, zero-filled outside the tensors), narrow
    // transformed operands through registers, wide transformed operands by rewriting the tile the
    // TMA producer (warp 0) landed; then they publish the stage to the MMA warp.  (TMA tile loads cost ~7-16 cycles per box ROW whatever its width:
    // with 32-96-byte rows of the narrow operands the TMA unit, not HBM, bounded every GEMM.)
    asm volatile("setmaxnreg.inc.sync.aligned.u32 152;");
    const int nxt = p.wg2x ? 256 : 128;
    const int t = warp >= 12 ? threadIdx.x - 384 : threadIdx.x - 256 + 128;
    const int G = p.lgroup;                       // warps sharing a stage (rows split G ways)
    const int NW = (nxt >> 5) / G, lw = (t >> 5) / G, ls = (t >> 5) % G, ln = t & 31;
    const int Ca = (kXform && p.a_xform) ? (kAmn ? p.M : p.K) : 0;
    const int Cb = (kXform && p.b_xform) ? (kBmn ? p.N : p.K) : 0;
    float* xa = s_coef + (kEpi == 1 ? 4 * p.N : 0);
    float* xb = xa + 3 * Ca;
    if (use_x) {
      // coefficient tables in smem: A: [scale|shift|scale2] x Ca, then B likewise
      for (int i = t; i < Ca; i += nxt) {
        xa[i] = p.a_scale[i];
        xa[Ca + i] = p.a_shift[i];
        xa[2 * Ca + i] = p.a_xform == 2 ? p.a_scale2[i] : 0.f;
      }
      for (int i = t; i < Cb; i += nxt) {
        xb[i] = p.b_scale[i];
        xb[Cb + i] = p.b_shift[i];
        xb[2 * Cb + i] = p.b_xform == 2 ? p.b_scale2[i] : 0.f;
      }
      named_bar_sync(2, nxt);
    }
    const ActParam apa = make_act((kXform && p.a_xform == 1) ? p.a_act : ACT_NONE);
    const ActParam apb = make_act((kXform && p.b_xform == 1) ? p.b_act : ACT_NONE);
    const int na = kAmn ? 2 : 1;                                         // panels of A
    const int nb = kBmn ? (kBN + 63) / 64 : (kBN + 127) / 128;  // panels of B

    // (tile, k-block) cursor over this CTA's work
    struct Cur { int w, kb, kb1, m_blk, n_blk; };
    const bool simple_work = p.ksplit == 1 && p.n_blocks == 1;   // one work item = one m-block
    auto cur_set = [&](Cur& c) {
      if (c.w < p.num_work) {
        if (simple_work) {
          c.m_blk = c.w; c.n_blk = 0; c.kb = 0; c.kb1 = p.num_k_blocks;
        } else {
          const int mn = c.w / p.ksplit, slab = c.w % p.ksplit;
          c.m_blk = mn / p.n_blocks; c.n_blk = mn % p.n_blocks;
          c.kb = slab * p.kb_per_split;
          c.kb1 = min(c.kb + p.kb_per_split, p.num_k_blocks);
        }
      }
    };
    auto cur_next = [&](Cur& c) {
      if (++c.kb >= c.kb1) { c.w += gridDim.x; cur_set(c); }
    };
    // geometry of panel pi (A panels first, then B) of the k-block at cursor c
    struct Pan { uint32_t off; int rows, row0, col0, rlimit, climit, logR, cshift; bool isA, mn; };
    auto panel_of = [&](const Cur& c, int pi) {
      Pan g;
      g.isA = pi < na;
      const int q = g.isA ? pi : pi - na;
      g.mn = g.isA ? (kAmn != 0) : (kBmn != 0);
      g.off = (g.isA ? 0u : (uint32_t)p.a_bytes) + (uint32_t)q * (g.mn ? kPanelBytes64 : 128 * 128);
      g.logR = g.mn ? 6 : 7;
      if (!g.mn) {  // K-major: rows are M (A) or N (B), channels along K
        g.row0 = g.isA ? c.m_blk * kBlockM : c.n_blk * kBN + q * 128;
        g.col0 = c.kb * kBlockK; g.climit = p.K;
        g.rlimit = g.isA ? min(128, p.M - g.row0)
                         : min(128, min(kBN - q * 128, p.N - g.row0));
        g.rows = g.rlimit;     // rows past the limit only feed outputs that are never stored
      } else {      // MN-major: rows are K (pixels), 64 channels of M/N per panel
        g.row0 = c.kb * kBlockK;
        g.col0 = (g.isA ? c.m_blk * kBlockM : c.n_blk * kBN) + q * 64;
        g.climit = g.isA ? p.M : p.N;
        g.rlimit = g.col0 < g.climit ? min(64, p.K - g.row0) : 0;
        // rows past K must read as zero (they are accumulated); a panel wholly past M / N only
        // feeds outputs that are never stored: leave it alone
        g.rows = g.col0 < g.climit ? 64 : 0;
      }
      if (g.rlimit < 0) g.rlimit = 0;
      if (g.rows < 0) g.rows = 0;
      // 16-byte chunk slots per row that the MMA can read: narrow operands (K or C <= 32) take
      // 2 or 4 lanes per row instead of 8
      int ncs = (g.climit - g.col0 + 7) >> 3;
      if (!g.mn) ncs = (ncs + 1) & ~1;   // K-steps of 16 columns: the odd chunk must read as zero
      g.cshift = ncs <= 2 ? 1 : (ncs <= 4 ? 2 : 3);
      // the last k-block of a longer K reuses a stage that full k-blocks wrote: all 8 chunks of
      // its rows are rewritten, those past K as zero (the MMA reads all 64 columns)
      if (!g.mn && p.num_k_blocks > 1) g.cshift = 3;
      return g;
    };
    // cp.async one panel (coalesced: 8 consecutive threads fetch the 128 bytes of one row)
    auto load_panel = [&](uint32_t dst, const __nv_bfloat16* src, long long ld, const Pan& g) {
      const int rpw = ((1 << g.logR) / G);          // rows of the panel per warp of the group
      const int rend = min(g.rows, (ls + 1) * rpw);
      const int total = rend << g.cshift;
      const __nv_bfloat16* base = src + (long long)g.row0 * ld + g.col0;
#pragma unroll 4
      for (int i = ((ls * rpw) << g.cshift) + ln; i < total; i += 32) {
        const int r = i >> g.cshift, lc = i & ((1 << g.cshift) - 1);
        const bool ok = r < g.rlimit && g.col0 + lc * 8 < g.climit;
        const __nv_bfloat16* sp = ok ? base + (long long)r * ld + lc * 8 : src;
        cp_async_zfill16(dst + (uint32_t)(r * 128 + ((lc ^ (r & 7)) << 4)), sp, ok ? 16 : 0);
      }
    };
    auto issue = [&](const Cur& c, int stage, int rnd) {
      gemm_wait(&bars->empty[stage], (rnd & 1) ^ 1);
      const uint32_t sA = smem_u32(smem + (size_t)stage * p.stage_bytes);
      for (int pi = 0; pi < na + nb; ++pi) {
        const Pan g = panel_of(c, pi);
        if (kXform && (g.isA ? p.a_xform : p.b_xform) != 0) continue;   // register path (consume)
        load_panel(sA + g.off, g.isA ? p.gA : p.gB, g.isA ? p.lda : p.ldb, g);
      }
    };
    auto consume = [&](const Cur& c, int stage, int rnd) {
      if (kXform && use_x) {
        const uint32_t sA = smem_u32(smem + (size_t)stage * p.stage_bytes);
        // narrow transformed operands: registers (few bytes per row, latency hidden by the batch)
#pragma unroll 1
        for (int pi = 0; pi < na + nb; ++pi) {
          const Pan g = panel_of(c, pi);
          const int mode = g.isA ? p.a_xform : p.b_xform;
          if (mode == 0 || (g.isA ? p.a_tma : p.b_tma)) continue;
          const ActParam& ap = g.isA ? apa : apb;
          const float* tab = g.isA ? xa : xb;
          const int Ct = g.isA ? Ca : Cb;
          const uint32_t t_s = smem_u32(tab), t_b = smem_u32(tab + Ct), t_s2 = smem_u32(tab + 2 * Ct);
          const float* gate = (mode == 1 && (g.mn || g.isA)) ? (g.isA ? p.a_gate : p.b_gate) : nullptr;
          const __nv_bfloat16* g1 = (g.isA ? p.gA : p.gB) + (long long)g.row0 * (g.isA ? p.lda : p.ldb);
          const __nv_bfloat16* g2 = mode == 2
              ? (g.isA ? p.gA2 : p.gB2) + (long long)g.row0 * (g.isA ? p.lda2 : p.ldb2) : g1;
          if (mode == 2)
            gxform_panel<2, false>(sA + g.off, 0u, g1, g.isA ? p.lda : p.ldb, g2, g.isA ? p.lda2 : p.ldb2,
                                   ls * ((1 << g.logR) / G), min(g.rows, (ls + 1) * ((1 << g.logR) / G)), g.rlimit, ln, g.cshift, ap, t_s, t_b, t_s2, g.col0, g.climit, gate,
                                   (unsigned)g.row0, (unsigned)p.gate_rps);
          else
            gxform_panel<1, false>(sA + g.off, 0u, g1, g.isA ? p.lda : p.ldb, g2, g.isA ? p.lda2 : p.ldb2,
                                   ls * ((1 << g.logR) / G), min(g.rows, (ls + 1) * ((1 << g.logR) / G)), g.rlimit, ln, g.cshift, ap, t_s, t_b, t_s2, g.col0, g.climit, gate,
                                   (unsigned)g.row0, (unsigned)p.gate_rps);
        }
        // wide transformed operands: the TMA producer loaded them; rewrite the tile in place
        if (p.a_tma || p.b_tma) {
          gemm_wait(&bars->xdone[stage], rnd & 1);
#pragma unroll 1
          for (int pi = 0; pi < na + nb; ++pi) {
            const Pan g = panel_of(c, pi);
            const int mode = g.isA ? p.a_xform : p.b_xform;
            if (mode == 0 || !(g.isA ? p.a_tma : p.b_tma)) continue;
            const ActParam& ap = g.isA ? apa : apb;
            const float* tab = g.isA ? xa : xb;
            const int Ct = g.isA ? Ca : Cb;
            const uint32_t t_s = smem_u32(tab), t_b = smem_u32(tab + Ct), t_s2 = smem_u32(tab + 2 * Ct);
            const float* gate = (mode == 1 && (g.mn || g.isA)) ? (g.isA ? p.a_gate : p.b_gate) : nullptr;
            const uint32_t op2 = sA + (g.isA ? p.a2_off : p.b2_off) +
                                 (g.off - (g.isA ? 0u : (uint32_t)p.a_bytes));
            // rows the TMA zero-filled (outside the tensor) must stay zero: limit = rlimit
            if (mode == 2)
              gxform_panel<2, true>(sA + g.off, op2, nullptr, 0, nullptr, 0, ls * ((1 << g.logR) / G),
                                    min(g.rlimit, (ls + 1) * ((1 << g.logR) / G)), g.rlimit, ln, 3, ap,
                                    t_s, t_b, t_s2, g.col0, g.climit, gate, (unsigned)g.row0,
                                    (unsigned)p.gate_rps);
            else
              gxform_panel<1, true>(sA + g.off, op2, nullptr, 0, nullptr, 0, ls * ((1 << g.logR) / G),
                                    min(g.rlimit, (ls + 1) * ((1 << g.logR) / G)), g.rlimit, ln, 3, ap,
                                    t_s, t_b, t_s2, g.col0, g.climit, gate, (unsigned)g.row0,
                                    (unsigned)p.gate_rps);
          }
        }
      }
      cp_async_wait<0>();
      fence_proxy_async_smem();
      __syncwarp();
      if (ln == 0) mbar_arrive(&bars->full[stage]);
    };

    // One loader WARP fills a whole stage, and every stage has ONE owner warp (stage s belongs to
    // warp s mod NW): the owner walks the rounds of its stage in order, so a parity wait on
    // empty[s] can never alias a phase two rounds away.  Each warp has a single stage in flight, so
    // the proxy fence before publishing it (a MEMBAR that waits for ALL of the thread's
    // outstanding cp.async) never waits for younger copies; the CTA has min(NW, S) stages in flight.
    Cur c;
    c.w = blockIdx.x;
    cur_set(c);
    // n = running k-block index, st = n % S, rnd = n / S (no divisions in the loop)
    int st = 0, rnd = 0;
    for (; c.w < p.num_work; cur_next(c)) {
      if (st % NW == lw) {
        issue(c, st, rnd);
        cp_async_commit();
        consume(c, st, rnd);
      }
      if (++st == S) { st = 0; ++rnd; }
    }
  }

  // ---- teardown ---------------------------------------------------------------------------------
  __syncthreads();
  if (p.has_bnf) {
    if (publish_partials(s_stats, p.N, p.bnf.partials, p.bnf.counter)) {
      bn_fwd_finalize(p.bnf, p.N);
      __syncthreads();
      if (threadIdx.x == 0) *p.bnf.counter = 0;
    }
  } else if (p.has_bnb) {
    if (publish_partials(s_stats, p.N, p.bnb.partials, p.bnb.counter)) {
      bn_bwd_finalize(p.bnb, p.N);
      __syncthreads();
      if (threadIdx.x == 0) *p.bnb.counter = 0;
    }
  }
}

// D[m][n] += the split-K partial tiles of (m, n), added in slab order
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ part, float* D,
                                                            long long ldd, int M, int N, int block_n,
                                                            int n_blocks, int ksplit) {
  const long long total = (long long)M * N;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int m = (int)(i / N), n = (int)(i % N);
    const int mn = (m / kBlockM) * n_blocks + n / block_n;
    const float* pp = part + (size_t)mn * ksplit * (kBlockM * kMaxBlockN) + (m % kBlockM) * kMaxBlockN + n % block_n;
    float acc = 0.f;
    for (int k = 0; k < ksplit; ++k) acc += __ldcg(pp + (size_t)k * (kBlockM * kMaxBlockN));
    D[(size_t)m * ldd + n] += acc;
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static int make_map_2d(CUtensorMap* map, const void* ptr, uint64_t inner, uint64_t outer,
                       uint64_t ld_elems, uint32_t box_inner, uint32_t box_outer) {
  static PFN_encodeTiled encode = get_encode_tiled();
  if (!encode) return set_error(YAMB_ECUDA, "cuTensorMapEncodeTiled entry point not found");
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld_elems * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (strides[0] & 15))
    return set_error(YAMB_EINVAL, "TMA operand must be 16-byte aligned with a 16-byte row pitch");
  CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims,
                      strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(YAMB_ECUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return 0;
}

// block_n is the wgmma width: 16, 32 or 64.  The 128 x block_n fp32 accumulator of a tile lives in
// the registers of one consumer warpgroup, and the kernel's 512 threads get at most 128 registers
// each, so wider tiles would spill.  An MN-major B is read in 64-column panels.
static int pick_block_n(int N, bool b_mn) {
  if (b_mn || N > 32) return 64;   // several n-blocks: 64 columns each, one staging sub-tile
  return N <= 16 ? 16 : 32;
}

// Launch of one instantiation: 0 or a YAMB_* code with the message set.
using LaunchFn = int (*)(int, int, cudaStream_t, const CUtensorMap&, const CUtensorMap&,
                         const CUtensorMap&, const CUtensorMap&, const CUtensorMap&, const GemmDev&);
template <bool XF, int EP, int BN, int AMN, int BMN>
static int launch_tc(int grid, int smem, cudaStream_t stream, const CUtensorMap& tmA,
                     const CUtensorMap& tmB, const CUtensorMap& tmA2, const CUtensorMap& tmB2,
                     const CUtensorMap& tmD, const GemmDev& p) {
  int rc = smem_optin("gemm launch", (const void*)gemm_tc_kernel<XF, EP, BN, AMN, BMN>, smem);
  if (rc) return rc;
  gemm_tc_kernel<XF, EP, BN, AMN, BMN><<<grid, 512, smem, stream>>>(tmA, tmB, tmA2, tmB2, tmD, p);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "gemm launch: %s", cudaGetErrorString(e));
  return 0;
}
template <int EP, int BN, int AMN, int BMN>
static LaunchFn pick_tc(bool xf) {
  return xf ? &launch_tc<true, EP, BN, AMN, BMN> : &launch_tc<false, EP, BN, AMN, BMN>;
}

// What a launch decides before it looks at a pointer: the argument checks, the tile grid and
// split-K, the warp roles, the shared-memory layout and the kernel instantiation.
struct GemmPlan {
  GemmDev p;
  LaunchFn fn;
  int xf;          // XF of the instantiation fn launches
  int sms;         // SM count planned for
  int grid;
  int smem_total;
};

// 0 or a YAMB_* code with the message set.  num_sms <= 0: the current device's SM count.
static int gemm_plan(const yamb_gemm* a, int num_sms, GemmPlan& pl) {
  if (!a || a->M <= 0 || a->N <= 0 || a->K <= 0) return set_error(YAMB_EINVAL, "bad GEMM shape");
  if ((a->N % 8) || (a->a_mn_major ? (a->M % 8) : (a->K % 8)) || (a->b_mn_major ? 0 : (a->K % 8)))
    return set_error(YAMB_EINVAL, "GEMM channel dims must be multiples of 8 (M=%d N=%d K=%d)",
                     a->M, a->N, a->K);
  if (a->epi < 0 || a->epi > 2) return set_error(YAMB_EINVAL, "bad epilogue");
  const int dev_ctas = num_sms > 0 ? num_sms : max_ctas();
  if (dev_ctas <= 0) return set_error(YAMB_ENODEV, "no CUDA device");

  GemmDev& p = pl.p;
  memset(&p, 0, sizeof(p));
  p.M = a->M; p.N = a->N; p.K = a->K;
  p.a_mn = a->a_mn_major ? 1 : 0;
  p.b_mn = a->b_mn_major ? 1 : 0;
  p.block_n = pick_block_n(a->N, p.b_mn != 0);
  p.m_blocks = (a->M + kBlockM - 1) / kBlockM;
  p.n_blocks = (a->N + p.block_n - 1) / p.block_n;
  p.num_k_blocks = (a->K + kBlockK - 1) / kBlockK;
  p.epi = a->epi;
  p.a_xform = a->a_xform; p.a_act = a->a_act;
  p.b_xform = a->b_xform; p.b_act = a->b_act;
  p.a_scale = a->a_scale; p.a_shift = a->a_shift; p.a_scale2 = a->a_scale2;
  p.b_scale = a->b_scale; p.b_shift = a->b_shift; p.b_scale2 = a->b_scale2;
  if ((p.a_xform && (!a->a_scale || !a->a_shift)) || (p.b_xform && (!a->b_scale || !a->b_shift)))
    return set_error(YAMB_EINVAL, "operand transform without coefficients");
  if ((p.a_xform == 2 && (!a->A2 || !a->a_scale2)) || (p.b_xform == 2 && (!a->B2 || !a->b_scale2)))
    return set_error(YAMB_EINVAL, "two-source transform without second tensor");
  p.has_residual = (a->epi == 0 && a->residual) ? 1 : 0;
  // transform-heavy / epilogue-light launches give warps 8-11 to the transform
  // warps 8-11 load/transform instead of running a second epilogue warpgroup when the epilogue
  // is light relative to the operand work: split-K wgrad (no store at all) or a forward/dgrad
  // store of <= 192 columns fed by more than one k-block per tile
  p.wg2x = ((a->a_xform || a->b_xform) &&
            (a->epi == 2 || (a->epi == 0 && p.block_n <= 192 && p.num_k_blocks >= 2))) ? 1 : 0;
  p.a_gate = a->a_xform == 1 ? a->a_gate : nullptr;
  p.b_gate = a->b_xform == 1 ? a->b_gate : nullptr;
  p.gate_rps = a->gate_rows_per_sample > 0 ? a->gate_rows_per_sample : 1;
  if ((p.a_gate || p.b_gate) && a->gate_rows_per_sample <= 0)
    return set_error(YAMB_EINVAL, "gate without gate_rows_per_sample");
  if (p.b_gate && !p.b_mn) return set_error(YAMB_EINVAL, "b_gate needs an MN-major B (rows = pixels)");
  p.D = a->D; p.ldd = a->ldd;
  if (a->epi == 0 && a->bn_fwd) { p.bnf = *a->bn_fwd; p.has_bnf = 1; }
  if (a->epi == 1) {
    if (!a->H || !a->h_scale || !a->h_shift || !a->bn_bwd)
      return set_error(YAMB_EINVAL, "dz epilogue needs H, h_scale, h_shift, bn_bwd");
    p.bnb = *a->bn_bwd; p.has_bnb = 1;
    p.h_scale = a->h_scale; p.h_shift = a->h_shift; p.h_act = a->h_act;
  }
  // split-K only for the atomic epilogue
  const int mn_tiles = p.m_blocks * p.n_blocks;
  int ctas = dev_ctas;
  if (a->max_ctas > 0 && a->max_ctas < ctas) ctas = a->max_ctas;
  p.ksplit = 1;
  if (a->epi == 2) {
    int want = (2 * ctas + mn_tiles - 1) / mn_tiles;
    int maxsplit = (p.num_k_blocks + 3) / 4;
    p.ksplit = want < 1 ? 1 : (want > maxsplit ? maxsplit : want);
    if (p.ksplit < 1) p.ksplit = 1;
  }
  p.kb_per_split = (p.num_k_blocks + p.ksplit - 1) / p.ksplit;
  p.ksplit = (p.num_k_blocks + p.kb_per_split - 1) / p.kb_per_split;  // no empty slabs
  p.num_work = mn_tiles * p.ksplit;

  // ---- shared memory plan ----
  const int b_panels = (p.block_n + 63) / 64;
  p.b_bytes = p.b_mn ? b_panels * kPanelBytes64 : ((p.block_n * 128 + 1023) / 1024) * 1024;
  // an MN-major A of <= 64 channels has a single live panel: the second one (rows 64..127 of the
  // MMA, outputs that are never stored) may alias the B region, the stage shrinks by 8 KB
  p.a_bytes = (p.a_mn && a->M <= 64) ? kPanelBytes64 : kABytes;
  int stage = p.a_bytes + p.b_bytes;
  // wide transformed operands come in by TMA (128-byte box rows) and are rewritten in place, a
  // second source needs its own region; narrow ones are combined in registers on their way in
  p.a_tma = (p.a_xform != 0 && (p.a_mn ? a->M : a->K) >= 64) ? 1 : 0;
  p.b_tma = (p.b_xform != 0 && (p.b_mn ? a->N : a->K) >= 64) ? 1 : 0;
  // transformed operands: 4 (2) loader warps share a stage so that its transform latency is short;
  // plain GEMMs are bound by load latency: one warp per stage, as many stages in flight as warps
  p.a2_off = p.b2_off = 0;
  if (p.a_tma && p.a_xform == 2) { p.a2_off = stage; stage += kABytes; }
  if (p.b_tma && p.b_xform == 2) { p.b2_off = stage; stage += p.b_bytes; }
  p.stage_bytes = stage;
  const bool xf = p.a_xform || p.b_xform;
  const int Ca = p.a_xform ? (p.a_mn ? p.M : p.K) : 0;
  const int Cb = p.b_xform ? (p.b_mn ? p.N : p.K) : 0;
  int fixed = 0;
  // every epilogue warp stages its own 32 x 64 sub-tile: 2 buffers each unless smem is short
  // raw side rows (H of epi 1, the residual of epi 0), one 32-row tile per epilogue warp
  const int side_bytes = (a->epi == 1 || p.has_residual) ? kEpiWarps * kWarpOutBytes : 0;
  const int coef_bytes = ((a->epi == 1 ? 4 * p.N : 0) + 3 * Ca + 3 * Cb) * 4;
  const int stats_bytes = (p.has_bnf || p.has_bnb) ? 2 * p.N * (int)sizeof(stat_t) : 0;
  const int budget = 232448 - 2048;  // 227 KB minus the kernel's static shared memory
  int stages = 0, out_bytes = 0;
  for (p.out_bufs = 2; p.out_bufs >= 1; --p.out_bufs) {
    out_bytes = (a->epi == 2) ? 0 : p.out_bufs * kEpiWarps * kWarpOutBytes;
    fixed = out_bytes + side_bytes + ((coef_bytes + 15) & ~15) + ((stats_bytes + 15) & ~15) +
            (int)sizeof(Bars) + 64;
    stages = (budget - fixed) / p.stage_bytes;
    // one 64-column sub-tile per tile: a warp's next staging use is two tile periods away (the
    // warpgroups alternate tiles), a single buffer never waits — spend the 32 KB on stages
    const bool single_sub = p.block_n <= 64 && a->epi != 2;
    if (single_sub && p.out_bufs == 2 && stages < kMaxStages) continue;
    if (stages >= 3 || p.out_bufs == 1) break;
  }
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages < 2) return set_error(YAMB_EINVAL, "GEMM tile does not fit shared memory");
  p.num_stages = stages;
  // Throughput-bound launches (many k-blocks per CTA): one loader warp per stage, all warps on
  // different stages (measured on b3: 2 / 4 warps per stage are 10 / 40 % slower).  Latency-bound
  // launches (a handful of k-blocks per CTA: 7x7 / 14x14 layers, split-K tails): the spare warps
  // share a stage so that its load/transform latency, which then IS the kernel time, shrinks.
  {
    const int grid_est = p.num_work < ctas ? p.num_work : ctas;
    const long long iters = ((long long)(p.num_work + grid_est - 1) / grid_est) * p.kb_per_split;
    const int nlw = p.wg2x ? 8 : 4;
    p.lgroup = 1;
    while (p.lgroup < 4 && (long long)(nlw / (p.lgroup * 2)) >= iters) p.lgroup *= 2;
    // fewer stages than loader warps: the surplus warps would idle — let them share stages
    while (p.lgroup < 4 && nlw / (p.lgroup * 2) >= stages) p.lgroup *= 2;
  }
  int off = stages * p.stage_bytes;
  p.off_out = off; off += out_bytes;
  p.off_hside = off; off += side_bytes;
  p.off_coef = off; off += (coef_bytes + 15) & ~15;
  p.off_stats = off; off += (stats_bytes + 15) & ~15;
  p.off_bars = (off + 15) & ~15; off = p.off_bars + (int)sizeof(Bars);
  pl.smem_total = off;  // the extern array is declared 1024-aligned: no slack needed

  // the operand layouts the layers produce (an MN-major B always has block_n 64)
  LaunchFn fn = nullptr;
  if (a->epi == 0 && !p.a_mn && !p.b_mn)   // forward
    fn = p.block_n == 64 ? pick_tc<0, 64, 0, 0>(xf) : p.block_n == 32 ? pick_tc<0, 32, 0, 0>(xf)
                                                                      : pick_tc<0, 16, 0, 0>(xf);
  else if (a->epi == 0 && !p.a_mn)         // dgrad (+ residual)
    fn = pick_tc<0, 64, 0, 1>(xf);
  else if (a->epi == 1 && !p.a_mn && p.b_mn)   // dgrad + dz: plain A (dh3) or two-source A, one
    fn = &launch_tc<true, 1, 64, 0, 1>;        // variant (XF = false spills 68 B at 128 registers)
  else if (a->epi == 2 && p.a_mn && p.b_mn)    // wgrad
    fn = pick_tc<2, 64, 1, 1>(xf);
  if (!fn)
    return set_error(YAMB_EINVAL, "GEMM operand layout not supported (epi %d, A %s, B %s)", a->epi,
                     p.a_mn ? "MN-major" : "K-major", p.b_mn ? "MN-major" : "K-major");
  pl.fn = fn;
  pl.xf = (a->epi == 1 || xf) ? 1 : 0;
  pl.sms = dev_ctas;
  pl.grid = p.num_work < ctas ? p.num_work : ctas;
  return 0;
}

int gemm_plan_query(const yamb_gemm* a, int num_sms, yamb_gemm_plan_info* out) {
  if (!out) return set_error(YAMB_EINVAL, "no plan output");
  GemmPlan pl;
  const int rc = gemm_plan(a, num_sms, pl);
  if (rc) return rc;
  const GemmDev& p = pl.p;
  memset(out, 0, sizeof(*out));
  out->xf = pl.xf; out->epi = p.epi; out->block_n = p.block_n; out->a_mn = p.a_mn; out->b_mn = p.b_mn;
  out->m_blocks = p.m_blocks; out->n_blocks = p.n_blocks; out->num_k_blocks = p.num_k_blocks;
  out->ksplit = p.ksplit; out->kb_per_split = p.kb_per_split; out->num_work = p.num_work;
  out->grid = pl.grid;
  out->a_tma = p.a_tma; out->b_tma = p.b_tma; out->wg2x = p.wg2x; out->lgroup = p.lgroup;
  out->num_stages = p.num_stages; out->out_bufs = p.out_bufs; out->smem_bytes = pl.smem_total;
  // the kernel's own rules (consumer warps, loader warps)
  out->reg_stats = (p.has_bnf || p.has_bnb) && p.n_blocks == 1;
  out->simple_work = p.ksplit == 1 && p.n_blocks == 1;
  return 0;
}

int gemm_launch(const yamb_gemm* a, cudaStream_t stream) {
  GemmPlan pl;
  int rc = gemm_plan(a, 0, pl);
  if (rc) return rc;
  GemmDev& p = pl.p;

  // ---- tensor maps ----
  CUtensorMap tmA, tmB, tmA2, tmB2, tmD;
  memset(&tmA, 0, sizeof(tmA)); memset(&tmB, 0, sizeof(tmB));
  memset(&tmA2, 0, sizeof(tmA2)); memset(&tmB2, 0, sizeof(tmB2));
  memset(&tmD, 0, sizeof(tmD));
  if (p.a_tma) {
    if (!p.a_mn) rc = make_map_2d(&tmA, a->A, a->K, a->M, a->lda, 64, 128);
    else rc = make_map_2d(&tmA, a->A, a->M, a->K, a->lda, 64, 64);
    if (rc) return rc;
    if (p.a_xform == 2) {
      if (!p.a_mn) rc = make_map_2d(&tmA2, a->A2, a->K, a->M, a->lda2, 64, 128);
      else rc = make_map_2d(&tmA2, a->A2, a->M, a->K, a->lda2, 64, 64);
      if (rc) return rc;
    }
  }
  if (p.b_tma) {
    if (!p.b_mn) rc = make_map_2d(&tmB, a->B, a->K, a->N, a->ldb, 64, p.block_n);
    else rc = make_map_2d(&tmB, a->B, a->N, a->K, a->ldb, 64, 64);
    if (rc) return rc;
    if (p.b_xform == 2) {
      if (!p.b_mn) rc = make_map_2d(&tmB2, a->B2, a->K, a->N, a->ldb2, 64, p.block_n);
      else rc = make_map_2d(&tmB2, a->B2, a->N, a->K, a->ldb2, 64, 64);
      if (rc) return rc;
    }
  }
  // operands are fetched with 16-byte cp.async: pointers 16-byte aligned, leading dims % 8 == 0
  {
    const void* ptrs[4] = {a->A, a->B, p.a_xform == 2 ? a->A2 : a->A, p.b_xform == 2 ? a->B2 : a->B};
    const long long lds[4] = {a->lda, a->ldb, p.a_xform == 2 ? a->lda2 : a->lda,
                              p.b_xform == 2 ? a->ldb2 : a->ldb};
    for (int i = 0; i < 4; ++i)
      if (!ptrs[i] || (reinterpret_cast<uintptr_t>(ptrs[i]) & 15) || (lds[i] % 8) || lds[i] <= 0)
        return set_error(YAMB_EINVAL, "GEMM operand %d: pointer must be 16-byte aligned, ld %% 8 == 0", i);
  }
  p.gA = (const __nv_bfloat16*)a->A; p.lda = a->lda;
  p.gB = (const __nv_bfloat16*)a->B; p.ldb = a->ldb;
  p.gA2 = (const __nv_bfloat16*)(p.a_xform == 2 ? a->A2 : nullptr); p.lda2 = a->lda2;
  p.gB2 = (const __nv_bfloat16*)(p.b_xform == 2 ? a->B2 : nullptr); p.ldb2 = a->ldb2;
  if (a->epi != 2) {
    rc = make_map_2d(&tmD, a->D, a->N, a->M, a->ldd, 64, 16);  // one warp's rows of a 64-row half
    if (rc) return rc;
  }
  if (a->epi == 1) { p.side = (const __nv_bfloat16*)a->H; p.lds = a->ldh; }
  else if (p.has_residual) { p.side = (const __nv_bfloat16*)a->residual; p.lds = a->ldr; }
  if (p.side && ((reinterpret_cast<uintptr_t>(p.side) & 15) || (p.lds % 8)))
    return set_error(YAMB_EINVAL, "side operand must be 16-byte aligned with lds % 8 == 0");

  cudaError_t e;
  if (a->epi == 2) {   // split-K partial tiles: released by the reduction below, on this stream
    rc = det_alloc((size_t)p.num_work * kBlockM * kMaxBlockN * sizeof(float), stream, &p.part);
    if (rc) return rc;
  }
  auto fail = [&](const char* what, cudaError_t err) {
    if (p.part) det_free(p.part, stream);
    return set_error(YAMB_ECUDA, "%s: %s", what, cudaGetErrorString(err));
  };
  if ((rc = pl.fn(pl.grid, pl.smem_total, stream, tmA, tmB, tmA2, tmB2, tmD, p))) {
    if (p.part) det_free(p.part, stream);
    return rc;
  }
  if (a->epi == 2) {
    const long long total = (long long)a->M * a->N;
    const long long cap = 4LL * pl.sms, blocks = (total + 255) / 256;
    splitk_reduce_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, stream>>>(
        p.part, reinterpret_cast<float*>(a->D), a->ldd, a->M, a->N, p.block_n, p.n_blocks, p.ksplit);
    e = cudaGetLastError();
    if (e != cudaSuccess) return fail("split-K reduce launch", e);
    rc = det_free(p.part, stream);
    if (rc) return rc;
  }
  return 0;
}

}  // namespace yamb
