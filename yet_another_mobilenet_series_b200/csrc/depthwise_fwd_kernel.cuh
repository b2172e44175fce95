// The depthwise forward kernel (see depthwise.cuh), included there twice: with YAMB_DW_GROUPED 0
// as the __global__ dw_fwd_kernel(DwFwdDev), with YAMB_DW_GROUPED 1 as the device function
// dw_fwd_body(p, vbid, vnblk) that one CTA of a grouped launch (depthwise_grouped.cu) runs as CTA
// vbid of a grid of vnblk.  Preprocessor text rather than a shared device function, so that
// dw_fwd_kernel keeps exactly the code it compiled to before the grouped launch existed: its
// block index, grid size and arrival count are the tokens blockIdx.x / gridDim.x / arrive_last
// they always were.  No include guard: meant to be included more than once.
// Forward, v4: the raw bf16 input tile (with halo) of tile t+1 streams into shared memory with
// cp.async (zero-fill outside the image) while tile t is transformed IN PLACE (BN + activation,
// rounded to bf16 like every other materialised activation) and convolved.
template <int K, int S, int CT, int TW>
#if YAMB_DW_GROUPED
__device__ __forceinline__ void dw_fwd_body(const DwFwdDev& p, const unsigned vbid,
                                            const unsigned vnblk) {
#else
__global__ void __launch_bounds__(256, (K == 3 ? kDw3MinBlocks : 1)) dw_fwd_kernel(
    const __grid_constant__ DwFwdDev p) {
#endif
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
  const unsigned t_end = (unsigned)(((unsigned long long)(YAMB_DW_BID + 1) * p.num_tiles) / YAMB_DW_NBLK);
  unsigned t = (unsigned)(((unsigned long long)YAMB_DW_BID * p.num_tiles) / YAMB_DW_NBLK);
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
    if (YAMB_DW_ARRIVE_LAST(p.bn.counter)) {
      bn_fwd_finalize(p.bn, p.C);
      __syncthreads();
      if (threadIdx.x == 0) *p.bn.counter = 0;
    }
  }
}
