// The depthwise backward kernel (see depthwise.cuh), included there twice: with YAMB_DW_BWD_SE 0
// as dw_bwd_kernel(DwBwdDev), with YAMB_DW_BWD_SE 1 as dw_bwd_se_kernel(DwBwdSeDev), the backward
// of the depthwise of a Squeeze-and-Excitation block.  There the staged dz is dY = d(a2 * gate), and
// each vector becomes dz = bf16((dY * gate[n][c] + dpool[n][c]) * act'(scale * h + shift)) (se_dz)
// before dh is formed from it.  Both come from one text so that they cannot drift apart, and as
// preprocessor text rather than a shared device function so that dw_bwd_kernel keeps exactly the
// code it compiled to before the SE variant existed (a function boundary changes its register
// allocation).  depthwise_grouped.cu includes it a third time, with YAMB_DW_GROUPED 1, as the
// device function dw_bwd_body(p, vbid, vnblk) that one CTA of a grouped launch runs as CTA vbid of
// a grid of vnblk (YAMB_DW_BID / YAMB_DW_NBLK / YAMB_DW_ARRIVE_LAST, see depthwise.cuh).  No
// include guard: meant to be included more than once.
template <int K, int S, int CT, int TAP0, int TAP1, bool DGRAD>
#if YAMB_DW_GROUPED
__device__ __forceinline__ void dw_bwd_body(const DwBwdDev& p, const unsigned vbid,
                                            const unsigned vnblk) {
#elif YAMB_DW_BWD_SE
__global__ void __launch_bounds__(256, (K == 3 ? kDw3MinBlocks : 1)) dw_bwd_se_kernel(
    const __grid_constant__ DwBwdSeDev pse) {
  const DwBwdDev& p = pse.dw;
#else
__global__ void __launch_bounds__(256, (K == 3 ? kDw3MinBlocks : 1)) dw_bwd_kernel(
    const __grid_constant__ DwBwdDev p) {
#endif
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
      if (c < p.C && g != 0.f) p.part[((size_t)YAMB_DW_BID * p.C + c) * KK + tp] = g;   // once per CTA
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
        cp_async_zfill16(d_dz + k * PSTEP * CT * 2, gdz + o, ok ? 16 : 0);
        cp_async_zfill16(d_h + k * PSTEP * CT * 2, gh + o, ok ? 16 : 0);
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
        cp_async_zfill16(d_x + k * PSTEP * CT * 2, gx + o, ok ? 16 : 0);
    }
    return mask;
  };

  // contiguous tile range per CTA (halo reuse in L2, see the forward kernel)
  const unsigned t_end = (unsigned)(((unsigned long long)(YAMB_DW_BID + 1) * p.num_tiles) / YAMB_DW_NBLK);
  unsigned t = (unsigned)(((unsigned long long)YAMB_DW_BID * p.num_tiles) / YAMB_DW_NBLK);
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
#if YAMB_DW_BWD_SE
          const uint4 rh = *(q + REG_ELEMS / 8);
          const uint4 rdz = se_dz(*q, rh, pse.se, n, cbase + g8 * 8);
#else
          const uint4 rdz = *q;
          const uint4 rh = *(q + REG_ELEMS / 8);
#endif
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
    if (YAMB_DW_ARRIVE_LAST(p.bn.counter)) {
      bn_bwd_finalize(p.bn, p.C);
      __syncthreads();
      if (threadIdx.x == 0) *p.bn.counter = 0;
    }
  }
}

