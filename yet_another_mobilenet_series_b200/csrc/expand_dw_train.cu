// Training-mode expand + depthwise forward with the expanded tile recomputed from x
// (yamb_expand_dw_train_fwd, include/yamb200.h): the kTrain mode of the one-launch block kernel
// (block_eval.cuh).  The expand GEMM still stores h1 for the backward; this launch replaces the
// depthwise forward that reads it back.  Per tile: x tile (+halo) -> wgmma expand -> bf16 ->
// BatchNorm 1 + act as dw_fwd applies it on load -> k x k stencil in dw_fwd's tap order -> raw z2
// (bf16) -> h2, and BatchNorm 2's batch statistics.  No W3, no project, no grid-wide barrier.
#include "block_eval.cuh"

namespace yamb {

template <class G, bool LEAN>
static int launch_train(BlockEvalDev& p, const yamb_expand_dw_train* a, cudaStream_t st) {
  // ---- shared-memory plan (bytes from the 1024-aligned base): x tile, W1 slice, the stencil
  //      threads' statistics (red: sums and sums of squares [NRUN][64] each), a1 tile, tap tables,
  //      barriers, the CTA's BatchNorm-2 totals (double [2][Chid]); no W3, no project operand ----
  p.xpanel_bytes = (G::NPI * 128 + 1023) & ~1023;
  int off = p.KB * p.xpanel_bytes;
  p.off_w1 = off; off += p.KB * 8192;
  p.off_w3 = off;
  p.off_h2 = off; off += 2 * G::NRUN * 64 * 4;
  p.off_h1 = off; off += ((G::NPI * kH1Pitch) + 15) & ~15;
  p.off_tab = off; off += 2 * tab_floats(G::K) * 4;
  p.off_c3 = off;
  p.off_bars = (off + 15) & ~15; off = p.off_bars + 16;
  p.off_stat = off; off += 2 * p.Chid * (int)sizeof(stat_t);
  int smem = off;
  const int x_read_end = (p.KB - 1) * p.xpanel_bytes + G::NCH * 8192;   // last byte the expand MMA may touch
  if (smem < x_read_end) smem = x_read_end;
  const int groups = (p.N + G::TI - 1) / G::TI;
  p.tiles_h = (p.Ho + G::TOH - 1) / G::TOH;
  p.tiles_w = (p.Wo + G::TOW - 1) / G::TOW;
  if ((long long)groups * p.tiles_h * p.tiles_w > 0x7fffffffLL)
    return set_error(YAMB_EINVAL, "expand_dw_train: too many tiles");
  p.num_tiles = groups * p.tiles_h * p.tiles_w;
  CUtensorMap tmX, tmW1, tmW3;
  {
    const cuuint64_t dims[4] = {(cuuint64_t)p.Cin, (cuuint64_t)p.W, (cuuint64_t)p.H, (cuuint64_t)p.N};
    const cuuint64_t str[3] = {(cuuint64_t)p.Cin * 2, (cuuint64_t)p.W * p.Cin * 2,
                               (cuuint64_t)p.H * p.W * p.Cin * 2};
    const cuuint32_t box[4] = {64, (cuuint32_t)G::IW, (cuuint32_t)G::IH, (cuuint32_t)G::TI};
    int rc = make_map(&tmX, a->x, 4, dims, str, box);
    if (rc) return rc;
  }
  {
    const cuuint64_t dims[2] = {(cuuint64_t)p.Cin, (cuuint64_t)p.Chid};
    const cuuint64_t str[1] = {(cuuint64_t)p.Cin * 2};
    const cuuint32_t box[2] = {64, 64};
    int rc = make_map(&tmW1, a->w_expand, 2, dims, str, box);
    if (rc) return rc;
  }
  memset(&tmW3, 0, sizeof(tmW3));
  const void* kern = (const void*)block_eval_kernel<G, true, LEAN, kTrain, false>;
  int rc = smem_optin("expand_dw_train", kern, smem, nullptr, 256, /*max_carveout=*/true);
  if (rc) return rc;
  // one resident CTA per SM, as the eval kernels (the expand fragments and the stencil registers)
  const int cap = max_ctas();
  const int grid = p.num_tiles < cap ? p.num_tiles : cap;
  block_eval_kernel<G, true, LEAN, kTrain, false><<<grid, 256, smem, st>>>(tmX, tmW1, tmW3, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "expand_dw_train launch: %s", cudaGetErrorString(e));
  return 0;
}

template <class G>
static int launch_train_act(BlockEvalDev& p, const yamb_expand_dw_train* a, cudaStream_t st) {
  // relu / relu6 / none are clamps of the packed bf16 pair (dw_fwd's ActParam kind 0)
  const bool lean = a->act == YAMB_ACT_NONE || a->act == YAMB_ACT_RELU || a->act == YAMB_ACT_RELU6;
  return lean ? launch_train<G, true>(p, a, st) : launch_train<G, false>(p, a, st);
}

// argument checks (no device needed) and the launch-independent fields of p
static int expand_dw_train_setup(const yamb_expand_dw_train* a, BlockEvalDev& p) {
  if (!a) return set_error(YAMB_EINVAL, "null args");
  if (a->N <= 0 || a->H <= 0 || a->W <= 0) return set_error(YAMB_EINVAL, "expand_dw_train: bad shape");
  if (a->Cin <= 0 || a->Chid <= 0 || a->Cin % 8 || a->Chid % 8)
    return set_error(YAMB_EINVAL, "expand_dw_train: channel counts must be positive multiples of 8");
  if (a->Cin > 256) return set_error(YAMB_EINVAL, "expand_dw_train: Cin <= 256 (got %d)", a->Cin);
  if ((a->kernel != 3 && a->kernel != 5 && a->kernel != 7) || (a->stride != 1 && a->stride != 2))
    return set_error(YAMB_EINVAL, "expand_dw_train: depthwise k in {3,5,7}, stride 1 or 2 (got k=%d s=%d)",
                     a->kernel, a->stride);
  if (a->act < YAMB_ACT_NONE || a->act > YAMB_ACT_HSWISH)
    return set_error(YAMB_EINVAL, "expand_dw_train: unknown activation %d", a->act);
  if (a->ldh < a->Chid || a->ldh % 8)
    return set_error(YAMB_EINVAL, "expand_dw_train: ldh must be a multiple of 8 >= Chid (got %d)", a->ldh);
  if (!a->x || !a->w_expand || !a->bn1_scale || !a->bn1_shift || !a->w_dw || !a->h2 || !a->bn)
    return set_error(YAMB_EINVAL, "expand_dw_train: null pointer");
  if (!a->bn->partials || !a->bn->counter || !a->bn->scale || !a->bn->shift)
    return set_error(YAMB_EINVAL, "expand_dw_train: BatchNorm 2 needs partials, counter, scale and shift");
  if ((((uintptr_t)a->x) | ((uintptr_t)a->w_expand) | ((uintptr_t)a->h2)) & 15)
    return set_error(YAMB_EINVAL, "expand_dw_train: x, w_expand and h2 must be 16-byte aligned");
  if ((long long)a->N * a->H * a->W > 0x7fffffffLL / 2)
    return set_error(YAMB_EINVAL, "expand_dw_train: too many pixels");
  memset(&p, 0, sizeof(p));
  p.N = a->N; p.H = a->H; p.W = a->W;
  p.Ho = (a->H - 1) / a->stride + 1;
  p.Wo = (a->W - 1) / a->stride + 1;
  p.Cin = a->Cin; p.Chid = a->Chid;
  p.act = a->act;
  p.x = (const __nv_bfloat16*)a->x;
  p.wdw = a->w_dw;
  p.mode = kTrain;
  p.cs = 1;
  p.s1 = a->bn1_scale; p.t1 = a->bn1_shift;
  p.h2 = (__nv_bfloat16*)a->h2;
  p.ldh = a->ldh;
  p.bn2f = *a->bn;
  const int kpad = (a->Cin + 15) / 16 * 16;
  p.nks = kpad / 16;
  p.KB = (kpad + 63) / 64;
  p.NC = (a->Chid + 63) / 64;
  return 0;
}

int expand_dw_train_launch(const yamb_expand_dw_train* a, cudaStream_t st) {
  BlockEvalDev p;
  int rc = expand_dw_train_setup(a, p);
  if (rc) return rc;
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  // the eval kernels' tile plans of (k, stride): stride 1, k = 3 / 5: 7x16 unless two 7x7 images
  // per tile take fewer tiles
  auto tiles_of = [&](int toh, int tow, int ti) {
    return (long long)((p.Ho + toh - 1) / toh) * ((p.Wo + tow - 1) / tow) * ((a->N + ti - 1) / ti);
  };
  const bool wide16 = tiles_of(7, 16, 1) <= tiles_of(7, 7, 2);
  if (a->kernel == 3) {
    if (a->stride == 2) return launch_train_act<EvGeom<3, 2, 7, 7, 1, 2>>(p, a, st);
    return wide16 ? launch_train_act<EvGeom<3, 1, 7, 16, 1, 4>>(p, a, st)
                  : launch_train_act<EvGeom<3, 1, 7, 7, 2, 4>>(p, a, st);
  }
  if (a->kernel == 5) {
    if (a->stride == 2) return launch_train_act<EvGeom<5, 2, 6, 7, 1, 2>>(p, a, st);
    return wide16 ? launch_train_act<EvGeom<5, 1, 7, 16, 1, 4>>(p, a, st)
                  : launch_train_act<EvGeom<5, 1, 7, 7, 2, 4>>(p, a, st);
  }
  if (a->stride == 2) return launch_train_act<EvGeom<7, 2, 4, 7, 1, 2>>(p, a, st);
  return launch_train_act<EvGeom<7, 1, 7, 7, 1, 2>>(p, a, st);
}

}  // namespace yamb
