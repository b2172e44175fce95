// Lightweight non-local block (AutoNL) core on NHWC bf16 activations, sm_90a.
//
// Replaces, behind yamb_nl_gram / yamb_nl_rowmat (include/yamb200.h), the two einsums of
// Nonlocal.forward (reference models/mobilenet_base.py:158-173) and their autograd backward:
//
//   theta = l[:, :c],  phi = l_sub[:, :c],  g = l_sub          (l_sub = l[:, :, ::s, ::s])
//   f[n,p,j] = (W/H) * sum_i theta[n,p,i] * sum_q phi[n,q,i] * g[n,q,j]
//
// The reference picks between (theta phi^T) g and theta (phi^T g) by a MAC count (:164-170); the
// two are the same sum re-associated.  Here the channel matrix F = phi^T g  [c x C]  is ALWAYS
// formed first (yamb_nl_gram, fp32) — it is at most 80 x 320 for every AutoNL shape — and applied
// per pixel row (yamb_nl_rowmat), so no [HW x HW'] attention map ever exists.
//
// Backward (df = gradient of f, s = W/H):
//   dtheta = s * df F^T        dF = s * theta^T df        dphi = g dF^T        dg = phi dF
// i.e. one more gram (over all pixels, two different tensors) and three more row x matrix passes.
//
// These are tiny batched products (<= 1.3 M MACs per sample, c = 6..80, not multiples of 8):
// plain fp32 FMA kernels with the per-sample matrix in shared memory; no tensor cores.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "host_util.h"
#include "prims.cuh"

namespace yamb {

struct NlGramDev {
  int N, H, W, sub, Hs, Ws;
  const __nv_bfloat16* X; long long ldx; int I;
  const __nv_bfloat16* Y; long long ldy; int J;
  float alpha;
  int rows_per_cta;
  float* part;       // [row chunks][N][I][J] slabs (plain stores), G itself for one chunk
};

// pixel index (inside one sample) of the r-th row of the row set
__device__ __forceinline__ int nl_row_pixel(int r, int W, int sub, int Ws) {
  return sub == 1 ? r : (r / Ws) * sub * W + (r % Ws) * sub;
}

// part[chunk][n][i][j] = alpha * sum over the chunk's rows r of X[n, pix(r), i] * Y[n, pix(r), j]
// grid = (row chunks, N); the launcher adds the chunk slabs into G in chunk order
__global__ void __launch_bounds__(256) nl_gram_kernel(const __grid_constant__ NlGramDev p) {
  extern __shared__ __align__(16) unsigned char nl_smem[];
  const int R = p.rows_per_cta;
  const int I2 = (p.I + 1) & ~1;                    // X row padded to an even channel count
  __nv_bfloat16* sX = reinterpret_cast<__nv_bfloat16*>(nl_smem);          // [R][I2]
  __nv_bfloat16* sY = sX + (size_t)R * I2;                                // [R][J]
  const int n = blockIdx.y;
  const int rows_total = p.Hs * p.Ws;
  const int r0 = blockIdx.x * R;
  const int nr = min(R, rows_total - r0);
  const size_t img = (size_t)n * p.H * p.W;
  for (int e = threadIdx.x; e < nr * I2; e += 256) {
    const int r = e / I2, i = e % I2;
    const size_t pix = img + nl_row_pixel(r0 + r, p.W, p.sub, p.Ws);
    sX[e] = i < p.I ? p.X[pix * p.ldx + i] : __float2bfloat16(0.f);
  }
  for (int e = threadIdx.x; e < nr * (p.J / 2); e += 256) {
    const int r = e / (p.J / 2), j2 = e % (p.J / 2);
    const size_t pix = img + nl_row_pixel(r0 + r, p.W, p.sub, p.Ws);
    reinterpret_cast<uint32_t*>(sY)[e] =
        *reinterpret_cast<const uint32_t*>(p.Y + pix * p.ldy + 2 * j2);
  }
  __syncthreads();
  const int IP = I2 / 2, JP = p.J / 2;
  float* S = p.part + ((size_t)blockIdx.x * p.N + n) * p.I * p.J;   // this CTA's slab
  for (int w = threadIdx.x; w < IP * JP; w += 256) {
    const int ip = w / JP, jp = w % JP;            // consecutive threads: consecutive column pairs
    float a00 = 0.f, a01 = 0.f, a10 = 0.f, a11 = 0.f;
    const uint32_t* xr = reinterpret_cast<const uint32_t*>(sX) + ip;
    const uint32_t* yr = reinterpret_cast<const uint32_t*>(sY) + jp;
#pragma unroll 4
    for (int r = 0; r < nr; ++r) {
      const uint32_t xv = xr[(size_t)r * IP], yv = yr[(size_t)r * JP];
      const float x0 = bf16lo(xv), x1 = bf16hi(xv), y0 = bf16lo(yv), y1 = bf16hi(yv);
      a00 = fmaf(x0, y0, a00); a01 = fmaf(x0, y1, a01);
      a10 = fmaf(x1, y0, a10); a11 = fmaf(x1, y1, a11);
    }
    const int i = 2 * ip, j = 2 * jp;
    S[(size_t)i * p.J + j] = p.alpha * a00;
    S[(size_t)i * p.J + j + 1] = p.alpha * a01;
    if (i + 1 < p.I) {
      S[(size_t)(i + 1) * p.J + j] = p.alpha * a10;
      S[(size_t)(i + 1) * p.J + j + 1] = p.alpha * a11;
    }
  }
}

struct NlRowmatDev {
  int N, H, W, sub, Hs, Ws;
  const __nv_bfloat16* X; long long ldx; int K;
  const float* Mat; long long mat_stride, sk, so; int O;
  float alpha;
  const __nv_bfloat16* base; long long ldb; int O_copy;
  int accumulate;
  __nv_bfloat16* out; long long ldo;
  int rows_per_cta;
};

// out[n, pix(r), o] = (base | out | 0) + alpha * sum_k X[n, pix(r), k] * Mat[n](k, o),  o < O
// (O even); columns [O, O_copy) are copied from base.       grid = (row chunks, N)
__global__ void __launch_bounds__(256) nl_rowmat_kernel(const __grid_constant__ NlRowmatDev p) {
  extern __shared__ __align__(16) unsigned char nl_smem[];
  const int R = p.rows_per_cta;                     // even
  const int K2 = (p.K + 1) & ~1;
  float* sM = reinterpret_cast<float*>(nl_smem);                                   // [K][O]
  __nv_bfloat16* sX = reinterpret_cast<__nv_bfloat16*>(sM + (size_t)p.K * p.O);    // [R][K2]
  const int n = blockIdx.y;
  const int rows_total = p.Hs * p.Ws;
  const int r0 = blockIdx.x * R;
  const int nr = min(R, rows_total - r0);
  const size_t img = (size_t)n * p.H * p.W;
  const float* M = p.Mat + (size_t)n * p.mat_stride;
  for (int e = threadIdx.x; e < p.K * p.O; e += 256) {
    const int k = e / p.O, o = e % p.O;
    sM[e] = M[(size_t)k * p.sk + (size_t)o * p.so];
  }
  for (int e = threadIdx.x; e < R * K2; e += 256) {
    const int r = e / K2, k = e % K2;
    __nv_bfloat16 v = __float2bfloat16(0.f);
    if (r < nr && k < p.K)
      v = p.X[(img + nl_row_pixel(r0 + r, p.W, p.sub, p.Ws)) * p.ldx + k];
    sX[e] = v;
  }
  __syncthreads();
  const int OP = p.O / 2, RP = (nr + 1) / 2;
  for (int w = threadIdx.x; w < RP * OP; w += 256) {
    const int rp = w / OP, op = w % OP;
    const __nv_bfloat16* x0 = sX + (size_t)(2 * rp) * K2;
    const __nv_bfloat16* x1 = x0 + K2;
    const float2* m = reinterpret_cast<const float2*>(sM) + op;
    float a00 = 0.f, a01 = 0.f, a10 = 0.f, a11 = 0.f;
#pragma unroll 4
    for (int k = 0; k < p.K; ++k) {
      const float2 mv = m[(size_t)k * OP];
      const float u0 = __bfloat162float(x0[k]), u1 = __bfloat162float(x1[k]);
      a00 = fmaf(u0, mv.x, a00); a01 = fmaf(u0, mv.y, a01);
      a10 = fmaf(u1, mv.x, a10); a11 = fmaf(u1, mv.y, a11);
    }
    const float acc[2][2] = {{a00, a01}, {a10, a11}};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = 2 * rp + h;
      if (r >= nr) continue;
      const size_t pix = img + nl_row_pixel(r0 + r, p.W, p.sub, p.Ws);
      float v0 = p.alpha * acc[h][0], v1 = p.alpha * acc[h][1];
      uint32_t* dst = reinterpret_cast<uint32_t*>(p.out + pix * p.ldo + 2 * op);
      if (p.base) {
        const uint32_t b = *reinterpret_cast<const uint32_t*>(p.base + pix * p.ldb + 2 * op);
        v0 += bf16lo(b); v1 += bf16hi(b);
      } else if (p.accumulate) {
        const uint32_t b = *dst;
        v0 += bf16lo(b); v1 += bf16hi(b);
      }
      *dst = pack_bf16(v0, v1);
    }
  }
  // pass-through columns [O, O_copy) of base
  if (p.base && p.O_copy > p.O) {
    const int CP = (p.O_copy - p.O) / 2;
    for (int w = threadIdx.x; w < nr * CP; w += 256) {
      const int r = w / CP, c = p.O + 2 * (w % CP);
      const size_t pix = img + nl_row_pixel(r0 + r, p.W, p.sub, p.Ws);
      *reinterpret_cast<uint32_t*>(p.out + pix * p.ldo + c) =
          *reinterpret_cast<const uint32_t*>(p.base + pix * p.ldb + c);
    }
  }
}

static int nl_common(int N, int H, int W, int sub) {
  if (N <= 0 || H <= 0 || W <= 0 || sub <= 0) return set_error(YAMB_EINVAL, "nonlocal: bad shape");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  if (N > 65535) return set_error(YAMB_EINVAL, "nonlocal: N > 65535");
  return 0;
}

int nl_gram_launch(const yamb_nl_gram* a, cudaStream_t st) {
  if (!a) return set_error(YAMB_EINVAL, "null args");
  int rc = nl_common(a->N, a->H, a->W, a->sub);
  if (rc) return rc;
  if (!a->X || !a->Y || !a->G || a->I <= 0 || a->J <= 0 || (a->J % 2) || (a->ldy % 2) ||
      a->I > a->ldx || a->J > a->ldy)
    return set_error(YAMB_EINVAL, "nl_gram: I=%d J=%d (J and ldy must be even)", a->I, a->J);
  NlGramDev p;
  p.N = a->N; p.H = a->H; p.W = a->W; p.sub = a->sub;
  p.Hs = (a->H + a->sub - 1) / a->sub; p.Ws = (a->W + a->sub - 1) / a->sub;
  p.X = (const __nv_bfloat16*)a->X; p.ldx = a->ldx; p.I = a->I;
  p.Y = (const __nv_bfloat16*)a->Y; p.ldy = a->ldy; p.J = a->J;
  p.alpha = a->alpha;
  const int rows = p.Hs * p.Ws;
  const int I2 = (a->I + 1) & ~1;
  const long long n_out = (long long)a->N * a->I * a->J;
  int R = rows < 64 ? rows : 64;
  // more row chunks when the batch alone cannot fill the SMs, as long as their slabs stay small
  // next to the L2 (every chunk writes and the reduction reads back a full [N][I][J] slab)
  while (R > 16 && (long long)((rows + R - 1) / R) * a->N < 2LL * max_ctas() &&
         (long long)((rows + R / 2 - 1) / (R / 2)) * n_out * 4 <= (16LL << 20))
    R /= 2;
  p.rows_per_cta = R;
  const size_t smem = (size_t)R * (I2 + a->J) * 2;
  if (smem > 200 * 1024) return set_error(YAMB_EINVAL, "nl_gram: rows too wide for shared memory");
  if ((rc = smem_optin("nl_gram", (const void*)nl_gram_kernel, smem))) return rc;
  dim3 grid((rows + R - 1) / R, a->N);
  p.part = a->G;
  if (grid.x > 1 && (rc = det_alloc((size_t)grid.x * n_out * sizeof(float), st, &p.part))) return rc;
  nl_gram_kernel<<<grid, 256, smem, st>>>(p);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    if (p.part != a->G) det_free(p.part, st);
    return set_error(YAMB_ECUDA, "nl_gram: %s", cudaGetErrorString(e));
  }
  return p.part != a->G ? det_reduce_launch(p.part, (int)grid.x, n_out, a->G, st, false) : 0;
}

int nl_rowmat_launch(const yamb_nl_rowmat* a, cudaStream_t st) {
  if (!a) return set_error(YAMB_EINVAL, "null args");
  int rc = nl_common(a->N, a->H, a->W, a->sub);
  if (rc) return rc;
  if (!a->X || !a->Mat || !a->out || a->K <= 0 || a->O <= 0 || (a->O % 2) || (a->ldo % 2) ||
      a->K > a->ldx || a->O > a->ldo)
    return set_error(YAMB_EINVAL, "nl_rowmat: K=%d O=%d (O and ldo must be even)", a->K, a->O);
  if (a->base && ((a->ldb % 2) || (a->O_copy > a->O && ((a->O_copy - a->O) % 2))))
    return set_error(YAMB_EINVAL, "nl_rowmat: base pitch / pass-through width must be even");
  if (a->base && a->accumulate)
    return set_error(YAMB_EINVAL, "nl_rowmat: base and accumulate are exclusive");
  NlRowmatDev p;
  p.N = a->N; p.H = a->H; p.W = a->W; p.sub = a->sub;
  p.Hs = (a->H + a->sub - 1) / a->sub; p.Ws = (a->W + a->sub - 1) / a->sub;
  p.X = (const __nv_bfloat16*)a->X; p.ldx = a->ldx; p.K = a->K;
  p.Mat = a->Mat; p.mat_stride = a->mat_stride; p.sk = a->sk; p.so = a->so; p.O = a->O;
  p.alpha = a->alpha;
  p.base = (const __nv_bfloat16*)a->base; p.ldb = a->ldb; p.O_copy = a->base ? a->O_copy : 0;
  p.accumulate = a->accumulate;
  p.out = (__nv_bfloat16*)a->out; p.ldo = a->ldo;
  const int rows = p.Hs * p.Ws;
  const int K2 = (a->K + 1) & ~1;
  int R = 32;
  while (R > 8 && (long long)((rows + R - 1) / R) * a->N < 2LL * max_ctas()) R /= 2;
  p.rows_per_cta = R;
  const size_t smem = (size_t)a->K * a->O * 4 + (size_t)R * K2 * 2;
  if (smem > 220 * 1024) return set_error(YAMB_EINVAL, "nl_rowmat: %d x %d matrix exceeds shared memory", a->K, a->O);
  if ((rc = smem_optin("nl_rowmat", (const void*)nl_rowmat_kernel, smem))) return rc;
  dim3 grid((rows + R - 1) / R, a->N);
  nl_rowmat_kernel<<<grid, 256, smem, st>>>(p);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "nl_rowmat: %s", cudaGetErrorString(e));
  return 0;
}

}  // namespace yamb
