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

// The kernel texts read a CTA's block index, its grid size and its arrival on a statistics counter
// through these names: the launch's own here; depthwise_grouped.cu includes the texts again as
// device functions that run one virtual CTA of a grouped launch.
#define YAMB_DW_GROUPED 0
#define YAMB_DW_BID blockIdx.x
#define YAMB_DW_NBLK gridDim.x
#define YAMB_DW_ARRIVE_LAST(counter) arrive_last(counter)

#include "depthwise_fwd_kernel.cuh"

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
#undef YAMB_DW_GROUPED
#undef YAMB_DW_BID
#undef YAMB_DW_NBLK
#undef YAMB_DW_ARRIVE_LAST

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

// grids: size only — the grids of the two kernels (the second 0 unless KK == 7), nothing launched
template <int KK, int SS, int CC, typename Dev>
static int launch_bwd(const Dev& p0, size_t smem, long long tiles, cudaStream_t st,
                      int* grids = nullptr) {
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
  if (grids) {
    grids[0] = g0;
    grids[1] = g1;
    return 0;
  }
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


// The dispatch over (k, stride, channel tile[, tile width]) of the depthwise launches: 32 / 64-channel
// tiles in depthwise.cu, 8 / 16 in depthwise_narrow.cu; YAMB_ECUDA when the combination is not
// built.  With `grid` (forward: 1 int; backward: 2, the second kernel's 0 unless k == 7) they only
// size the launch — the grid every launch of that shape uses — and enqueue nothing.
int dw_fwd_dispatch(const DwFwdDev& p, int k, int s, int ct, int tw, size_t smem, cudaStream_t st,
                    int* grid = nullptr);
int dw_fwd_dispatch_narrow(const DwFwdDev& p, int k, int s, int ct, int tw, size_t smem,
                           cudaStream_t st, int* grid = nullptr);
int dw_bwd_dispatch(const DwBwdDev& p, int k, int s, int ct, size_t smem, cudaStream_t st,
                    int* grid = nullptr);
int dw_bwd_dispatch_narrow(const DwBwdDev& p, int k, int s, int ct, size_t smem, cudaStream_t st,
                           int* grid = nullptr);

// Check the arguments of a depthwise forward / backward and fill the kernel arguments, the channel
// tile (forward: and the tile width) and the dynamic shared memory (depthwise.cu): 0, YAMB_EINVAL,
// or YAMB_ENODEV without a device.  `check_device` false: every check but the device's (the
// grouped launcher validates all its branches before it asks for the device).
int dw_fwd_setup(const yamb_dw_fwd* a, DwFwdDev* p, int* ct, int* tw, size_t* smem,
                 bool check_device = true);
int dw_bwd_setup(const yamb_dw_bwd* a, DwBwdDev* p, int* ct, size_t* smem,
                 bool check_device = true);

// The dispatch over (k, stride, channel tile) of the SE depthwise backward: 32 / 64-channel tiles in
// depthwise_se.cu, 8 / 16 in depthwise_se_narrow.cu
int dw_bwd_se_dispatch(const DwBwdSeDev& p, int k, int s, int ct, size_t smem, cudaStream_t st);
int dw_bwd_se_dispatch_narrow(const DwBwdSeDev& p, int k, int s, int ct, size_t smem,
                              cudaStream_t st);

}  // namespace yamb
