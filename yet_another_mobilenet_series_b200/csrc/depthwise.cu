// Depthwise k x k convolution: host side and the 32 / 64-channel-tile instantiations
// (kernels: depthwise.cuh; 8 / 16-channel tiles: depthwise_narrow.cu).
#include "depthwise.cuh"

namespace yamb {

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
static int check_common(int N, int H, int W, int C, int ldc, int k, int stride) {
  if (N <= 0 || H <= 0 || W <= 0 || C <= 0) return set_error(YAMB_EINVAL, "depthwise: bad shape");
  if (C % 8 || ldc % 8 || C > ldc) return set_error(YAMB_EINVAL, "depthwise: C=%d ldc=%d", C, ldc);
  if (k != 3 && k != 5 && k != 7) return set_error(YAMB_EINVAL, "depthwise: k=%d", k);
  if (stride != 1 && stride != 2) return set_error(YAMB_EINVAL, "depthwise: stride=%d", stride);
  if (C > 4096) return set_error(YAMB_EINVAL, "depthwise: C > 4096 per slice");
  return 0;
}

// Channels per tile: 64, unless 32-channel tiles waste fewer padded channels (C = 96, 144: the
// widest early layers would run a quarter of their lanes on padding).  Branches of <= 16 channels
// (searched networks: AtomNAS keeps branches of 1-23 channels at 56 x 56, padded to 8 / 16 / 24)
// get 8- or 16-channel tiles — with 32-channel tiles three quarters / half of the lanes computed
// padding — as long as the image is tall enough for the 64- / 32-row tiles that go with them.
static int pick_ct(int C, int H) {
  if (C <= 8 && H >= 28) return 8;
  if (C <= 16 && H >= 14) return 16;
  if (C <= 32) return 32;
  const int pad64 = (C + 63) / 64 * 64, pad32 = (C + 31) / 32 * 32;
  return pad32 < pad64 ? 32 : 64;
}

int dw_fwd_launch(const yamb_dw_fwd* a, cudaStream_t st) {
  if (!a) return set_error(YAMB_EINVAL, "null args");
  int rc = check_common(a->N, a->H, a->W, a->C, a->ldc, a->k, a->stride);
  if (rc) return rc;
  if (!a->x || !a->y || !a->w) return set_error(YAMB_EINVAL, "depthwise fwd: null pointer");
  if ((((uintptr_t)a->x) | ((uintptr_t)a->y)) & 15)
    return set_error(YAMB_EINVAL, "depthwise: activations must be 16-byte aligned");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  const int k = a->k, s = a->stride, pad = (k - 1) / 2;
  const int ct = pick_ct(a->C, (a->H + 2 * pad - k) / s + 1);
  DwFwdDev p;
  p.N = a->N; p.H = a->H; p.W = a->W; p.C = a->C; p.ldc = a->ldc;
  p.Ho = (a->H + 2 * pad - k) / s + 1;
  p.Wo = (a->W + 2 * pad - k) / s + 1;
  p.x = (const __nv_bfloat16*)a->x; p.y = (__nv_bfloat16*)a->y;
  p.in_scale = a->in_scale; p.in_shift = a->in_shift; p.in_act = a->in_act;
  p.w = a->w;
  p.has_bn = a->bn ? 1 : 0;
  if (a->bn) p.bn = *a->bn;
  const int tw = (k == 7 || p.Wo <= 8) ? 1 : 2;
  const int toh = 512 / ct, tow = 8 * tw;   // (256 / (ct / 4) strips / 8 columns) x 4 rows
  p.tiles_h = (p.Ho + toh - 1) / toh;
  p.tiles_w = (p.Wo + tow - 1) / tow;
  p.chunks = (a->C + ct - 1) / ct;
  {
    long long nt = (long long)p.chunks * a->N * p.tiles_h * p.tiles_w;
    if (nt > 0x7fffffffLL) return set_error(YAMB_EINVAL, "depthwise: too many tiles");
    p.num_tiles = (int)nt;
  }
  const int ih = (toh - 1) * s + k, iw = (tow - 1) * s + k;
  const size_t smem = (size_t)ih * iw * ct * sizeof(float) + 2 * (size_t)ct * sizeof(stat_t);
  if (smem > 220 * 1024) return set_error(YAMB_EINVAL, "depthwise fwd: tile too large");
  if (ct <= 16) return dw_fwd_dispatch_narrow(p, k, s, ct, tw, smem, st);
#define YAMB_FWD_CASE(KK, SS, CC, TT) \
  if (k == KK && s == SS && ct == CC && tw == TT) return launch_k(dw_fwd_kernel<KK, SS, CC, TT>, p, smem, p.num_tiles, st)
  YAMB_FWD_CASE(3, 1, 64, 1); YAMB_FWD_CASE(3, 1, 64, 2); YAMB_FWD_CASE(3, 2, 64, 1); YAMB_FWD_CASE(3, 2, 64, 2);
  YAMB_FWD_CASE(3, 1, 32, 1); YAMB_FWD_CASE(3, 1, 32, 2); YAMB_FWD_CASE(3, 2, 32, 1); YAMB_FWD_CASE(3, 2, 32, 2);
  YAMB_FWD_CASE(5, 1, 64, 1); YAMB_FWD_CASE(5, 1, 64, 2); YAMB_FWD_CASE(5, 2, 64, 1); YAMB_FWD_CASE(5, 2, 64, 2);
  YAMB_FWD_CASE(5, 1, 32, 1); YAMB_FWD_CASE(5, 1, 32, 2); YAMB_FWD_CASE(5, 2, 32, 1); YAMB_FWD_CASE(5, 2, 32, 2);
  YAMB_FWD_CASE(7, 1, 64, 1); YAMB_FWD_CASE(7, 2, 64, 1); YAMB_FWD_CASE(7, 1, 32, 1); YAMB_FWD_CASE(7, 2, 32, 1);
#undef YAMB_FWD_CASE
  return set_error(YAMB_ECUDA, "dw fwd launch: no kernel for k=%d stride=%d ct=%d tw=%d", k, s, ct, tw);
}

int dw_bwd_launch(const yamb_dw_bwd* a, cudaStream_t st) {
  if (!a) return set_error(YAMB_EINVAL, "null args");
  int rc = check_common(a->N, a->H, a->W, a->C, a->ldc, a->k, a->stride);
  if (rc) return rc;
  if (!a->ca || !a->cb || !a->cc || !a->dz || !a->h || !a->x || !a->dx || !a->dw || !a->w)
    return set_error(YAMB_EINVAL, "depthwise bwd: null pointer");
  // dz, h and x stream into shared memory in 16-byte cp.async pieces; dx is stored and residual
  // read 4 channels (8 bytes) at a time
  if ((((uintptr_t)a->dz) | ((uintptr_t)a->h) | ((uintptr_t)a->x)) & 15)
    return set_error(YAMB_EINVAL, "depthwise bwd: dz, h and x must be 16-byte aligned");
  if ((((uintptr_t)a->dx) | ((uintptr_t)a->residual)) & 7)
    return set_error(YAMB_EINVAL, "depthwise bwd: dx and residual must be 8-byte aligned");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  const int k = a->k, s = a->stride, pad = (k - 1) / 2;
  const int ct = pick_ct(a->C, a->H);
  DwBwdDev p;
  p.N = a->N; p.H = a->H; p.W = a->W; p.C = a->C; p.ldc = a->ldc;
  p.Ho = (a->H + 2 * pad - k) / s + 1;
  p.Wo = (a->W + 2 * pad - k) / s + 1;
  p.dz = (const __nv_bfloat16*)a->dz; p.h = (const __nv_bfloat16*)a->h;
  p.ca = a->ca; p.cb = a->cb; p.cc = a->cc;
  p.w = a->w; p.dw = a->dw;
  p.x = (const __nv_bfloat16*)a->x;
  p.in_scale = a->in_scale; p.in_shift = a->in_shift; p.in_act = a->in_act;
  p.dx = (__nv_bfloat16*)a->dx;
  p.residual = (const __nv_bfloat16*)a->residual;
  p.has_bn = a->bn ? 1 : 0;
  if (a->bn) p.bn = *a->bn;
  const int tih = 512 / ct, tiw = 8;        // (256 / (ct / 4) spatial threads / 4) x 2 rows
  const int rh = s == 1 ? tih + k - 1 : (tih + k - 1) / 2 + 1;
  const int rw = s == 1 ? tiw + k - 1 : (tiw + k - 1) / 2 + 1;
  p.tiles_h = (a->H + tih - 1) / tih;
  p.tiles_w = (a->W + tiw - 1) / tiw;
  p.chunks = (a->C + ct - 1) / ct;
  {
    long long nt = (long long)p.chunks * a->N * p.tiles_h * p.tiles_w;
    if (nt > 0x7fffffffLL) return set_error(YAMB_EINVAL, "depthwise: too many tiles");
    p.num_tiles = (int)nt;
  }
  // two staging buffers of bf16 {dz, h over the region; x over the tile} + fp32 tables
  const size_t smem =
      ((size_t)(2 * rh * rw + tih * tiw) * ct + (size_t)(7 + 2 * k * k) * ct) * sizeof(float) +
      2 * (size_t)ct * sizeof(stat_t);
  if (smem > 220 * 1024) return set_error(YAMB_EINVAL, "depthwise bwd: slice too wide for smem");
  if (ct <= 16) rc = dw_bwd_dispatch_narrow(p, k, s, ct, smem, st);
  else if (k == 3 && s == 1 && ct == 64) YAMB_DW_BWD(3, 1, 64, p, smem, p.num_tiles, st);
  else if (k == 3 && s == 2 && ct == 64) YAMB_DW_BWD(3, 2, 64, p, smem, p.num_tiles, st);
  else if (k == 3 && s == 1) YAMB_DW_BWD(3, 1, 32, p, smem, p.num_tiles, st);
  else if (k == 3 && s == 2) YAMB_DW_BWD(3, 2, 32, p, smem, p.num_tiles, st);
  else if (k == 5 && s == 1 && ct == 64) YAMB_DW_BWD(5, 1, 64, p, smem, p.num_tiles, st);
  else if (k == 5 && s == 2 && ct == 64) YAMB_DW_BWD(5, 2, 64, p, smem, p.num_tiles, st);
  else if (k == 5 && s == 1) YAMB_DW_BWD(5, 1, 32, p, smem, p.num_tiles, st);
  else if (k == 5 && s == 2) YAMB_DW_BWD(5, 2, 32, p, smem, p.num_tiles, st);
  else if (k == 7 && s == 1 && ct == 64) YAMB_DW_BWD(7, 1, 64, p, smem, p.num_tiles, st);
  else if (k == 7 && s == 2 && ct == 64) YAMB_DW_BWD(7, 2, 64, p, smem, p.num_tiles, st);
  else if (k == 7 && s == 1) YAMB_DW_BWD(7, 1, 32, p, smem, p.num_tiles, st);
  else YAMB_DW_BWD(7, 2, 32, p, smem, p.num_tiles, st);
  return rc;
}

}  // namespace yamb
