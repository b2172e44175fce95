// Squeeze-and-Excitation fully connected layers on the pooled [N, C] vectors, sm_90a.
//
// Replaces, behind yamb_se_fc_fwd / yamb_se_fc_bwd (include/yamb200.h), the two 1x1 convolutions
// on [N, C, 1, 1] of SqueezeAndExcitation.forward and the sigmoid
// (reference models/mobilenet_base.py:110-113: se_reduce -> active_fn -> se_expand -> sigmoid) and
// their autograd backward, which round 1 left to ~12 ATen/cuBLAS launches per SE block:
//   forward : u = W_r s + b_r ;  v = act(u) ;  gate = sigmoid(W_e v + b_e)
//   backward: dt = dgate*gate*(1-gate) ;  du = (W_e^T dt) * act'(u) ;  dpool = (W_r^T du) / HW ;
//             dW_e += dt^T v, db_e += sum dt, dW_r += du^T s, db_r += sum du   (sums over samples)
// fp32 throughout (the reference keeps these tiny layers in fp32 too).  Every product is one launch
// of a small tiled SGEMM with the bias / activation / sigmoid / act' step as its epilogue.
// C <= 4096, R <= 1024.
#include <cuda_runtime.h>
#include <string.h>

#include "host_util.h"
#include "prims.cuh"

namespace yamb {

// ---- one small tiled fp32 GEMM for every product of the SE branch -----------------------------------
// C[m][n] = epilogue( sum_k A(m,k) * B(k,n) ),  A(m,k) = A[m*a_rs + k*a_cs], B(k,n) = B[k*b_rs + n*b_cs]
// (arbitrary strides: transposed operands cost nothing).  64 x 64 outputs per CTA, K in chunks of
// 16 staged in shared memory with coalesced loads, 4 x 4 outputs per thread.  The per-thread serial
// loops of the first version of these kernels (one dependent load batch per iteration, 14 warps per
// SM) ran 200 us per product at AtomNAS-C+ sizes; tiled, every product is a few microseconds.
struct SeGemm {
  int M, N, K;
  const float* A; long long a_rs, a_cs;
  const float* B; long long b_rs, b_cs;
  float* C; long long c_rs;          // C[m*c_rs + n]
  float alpha;
  int epi;                           // 0 store alpha*acc | 1 u=acc+bias: C=u, C2=act(u) | 2 C=sigmoid(acc+bias)
                                     // 3 C=acc*act'(E[m][n]) (+ column sums into colsum) | 4 C += acc
                                     // 5 atomicAdd(C, acc): split-K partial sums (grid.z slabs)
  int k_per_slab;                    // K range of one grid.z slab (epi 5), else K
  const float* bias;                 // [N]
  const float* E; long long e_rs;    // epi 3
  float* C2;                         // epi 1 second output, same layout as C
  float* colsum;                     // epi 3: colsum[n] += sum_m C[m][n]
  int act;
};

constexpr int kSgT = 64, kSgK = 16;

__global__ void __launch_bounds__(256) se_gemm_kernel(const __grid_constant__ SeGemm p) {
  __shared__ float sA[kSgK][kSgT + 4];
  __shared__ float sB[kSgK][kSgT + 4];
  __shared__ float s_col[kSgT];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * kSgT, n0 = blockIdx.x * kSgT;
  const int tm = (tid / 16) * 4, tn = (tid % 16) * 4;      // this thread's 4 x 4 outputs
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  // loader roles: 1024 elements per operand tile, 4 per thread; the unit-stride dimension runs
  // along consecutive threads
  const bool a_kfast = p.a_cs == 1, b_nfast = p.b_cs == 1;
  const int k_beg = blockIdx.z * p.k_per_slab, k_end = min(p.K, k_beg + p.k_per_slab);
  for (int k0 = k_beg; k0 < k_end; k0 += kSgK) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int e = tid + r * 256;
      int m, k;
      if (a_kfast) { k = e % kSgK; m = e / kSgK; } else { m = e % kSgT; k = e / kSgT; }
      float v = 0.f;
      if (m0 + m < p.M && k0 + k < k_end) v = p.A[(size_t)(m0 + m) * p.a_rs + (size_t)(k0 + k) * p.a_cs];
      sA[k][m] = v;
      int n, kb;
      if (b_nfast) { n = e % kSgT; kb = e / kSgT; } else { kb = e % kSgK; n = e / kSgK; }
      float w = 0.f;
      if (n0 + n < p.N && k0 + kb < k_end) w = p.B[(size_t)(k0 + kb) * p.b_rs + (size_t)(n0 + n) * p.b_cs];
      sB[kb][n] = w;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kSgK; ++k) {
      const float4 av = *reinterpret_cast<const float4*>(&sA[k][tm]);
      const float4 bv = *reinterpret_cast<const float4*>(&sB[k][tn]);
      const float am[4] = {av.x, av.y, av.z, av.w}, bn[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(am[i], bn[j], acc[i][j]);
    }
    __syncthreads();
  }
  if (p.epi == 3 && p.colsum) {
    if (tid < kSgT) s_col[tid] = 0.f;
    __syncthreads();
  }
  float csum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + tm + i;
    if (m >= p.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tn + j;
      if (n >= p.N) continue;
      float v = acc[i][j] * p.alpha;
      float* c = p.C + (size_t)m * p.c_rs + n;
      switch (p.epi) {
        case 1: { v += p.bias[n]; *c = v; p.C2[(size_t)m * p.c_rs + n] = act_fwd(v, p.act); break; }
        case 2: { v += p.bias[n]; *c = 1.f / (1.f + __expf(-v)); break; }
        case 3: { v *= act_bwd(p.E[(size_t)m * p.e_rs + n], p.act); *c = v; csum[j] += v; break; }
        case 4: *c += v; break;
        case 5: atomicAdd(c, v); break;
        default: *c = v;
      }
    }
  }
  if (p.epi == 3 && p.colsum) {
#pragma unroll
    for (int j = 0; j < 4; ++j) atomicAdd(&s_col[tn + j], csum[j]);
    __syncthreads();
    if (tid < kSgT && n0 + tid < p.N) atomicAdd(p.colsum + n0 + tid, s_col[tid]);
  }
}

static cudaError_t se_gemm(SeGemm g, cudaStream_t st, int ksplit = 1) {
  g.k_per_slab = ((g.K + ksplit - 1) / ksplit + kSgK - 1) / kSgK * kSgK;
  dim3 grid((g.N + kSgT - 1) / kSgT, (g.M + kSgT - 1) / kSgT, (g.K + g.k_per_slab - 1) / g.k_per_slab);
  se_gemm_kernel<<<grid, 256, 0, st>>>(g);
  return cudaGetLastError();
}

// K slabs for a product whose output is small and whose K is long (u, du: [N][R] with K = C):
// enough CTAs to fill the GPU, at least 4 k-chunks per slab
static int se_ksplit(int M, int N, int K) {
  const int tiles = ((M + kSgT - 1) / kSgT) * ((N + kSgT - 1) / kSgT);
  int want = (2 * max_ctas() + tiles - 1) / tiles;
  const int most = (K + 4 * kSgK - 1) / (4 * kSgK);
  if (want > most) want = most;
  return want < 1 ? 1 : want;
}

// finish of the split-K products:  u += b_r, v = act(u)   |   du = acc * act'(u), db_r += col sums
__global__ void __launch_bounds__(256) se_finish_kernel(int N, int R, float* u, float* v,
                                                        const float* b_r, const float* u_saved,
                                                        float* g_br, int act, int mode) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= R) return;
  const int n0 = blockIdx.y * 32, n1 = min(N, n0 + 32);
  float s = 0.f;
  for (int n = n0; n < n1; ++n) {
    const size_t i = (size_t)n * R + j;
    if (mode == 0) {
      const float x = u[i] + b_r[j];
      u[i] = x;
      v[i] = act_fwd(x, act);
    } else {
      const float d = u[i] * act_bwd(u_saved[i], act);   // here `u` is the du accumulator
      u[i] = d;
      s += d;
    }
  }
  if (mode == 1) atomicAdd(g_br + j, s);
}

// dt = dgate * gate * (1 - gate); g_be[c] += sum_n dt[n][c]     thread = channel, CTA = sample slab
__global__ void __launch_bounds__(256) se_dt_kernel(int N, int C, const float* dgate, const float* gate,
                                                    float* dt, float* g_be, int rows_per_cta) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= C) return;
  const int n0 = blockIdx.y * rows_per_cta, n1 = min(N, n0 + rows_per_cta);
  float s = 0.f;
  for (int n = n0; n < n1; ++n) {
    const float g = gate[(size_t)n * C + c];
    const float v = dgate[(size_t)n * C + c] * g * (1.f - g);
    dt[(size_t)n * C + c] = v;
    s += v;
  }
  atomicAdd(g_be + c, s);
}

static int se_fc_check(int N, int C, int R) {
  if (N <= 0 || C <= 0 || R <= 0 || C > 4096 || R > 1024)
    return set_error(YAMB_EINVAL, "se_fc: N=%d C=%d R=%d", N, C, R);
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  return 0;
}

int se_fc_fwd_launch(const yamb_se_fc* a, cudaStream_t st) {
  if (!a) return set_error(YAMB_EINVAL, "null args");
  int rc = se_fc_check(a->N, a->C, a->R);
  if (rc) return rc;
  if (!a->pooled || !a->w_r || !a->b_r || !a->w_e || !a->b_e || !a->u || !a->v || !a->gate)
    return set_error(YAMB_EINVAL, "se_fc: null pointer");
  SeGemm g;
  memset(&g, 0, sizeof(g));
  // u[N][R] = s[N][C] * W_r[R][C]^T + b_r ; v = act(u)
  g.M = a->N; g.N = a->R; g.K = a->C;
  g.A = a->pooled; g.a_rs = a->C; g.a_cs = 1;
  g.B = a->w_r; g.b_rs = 1; g.b_cs = a->C;
  g.C = a->u; g.c_rs = a->R; g.alpha = 1.f; g.epi = 5;
  cudaError_t e = cudaMemsetAsync(a->u, 0, (size_t)a->N * a->R * sizeof(float), st);
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "se_fc memset: %s", cudaGetErrorString(e));
  // deterministic: one K slab, so every u element is one atomicAdd onto the zeroed buffer
  e = se_gemm(g, st, a->deterministic ? 1 : se_ksplit(g.M, g.N, g.K));
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "se_fc fwd (reduce): %s", cudaGetErrorString(e));
  {
    dim3 fg((a->R + 255) / 256, (a->N + 31) / 32);
    se_finish_kernel<<<fg, 256, 0, st>>>(a->N, a->R, a->u, a->v, a->b_r, nullptr, nullptr, a->act, 0);
  }
  // gate[N][C] = sigmoid(v[N][R] * W_e[C][R]^T + b_e)
  memset(&g, 0, sizeof(g));
  g.M = a->N; g.N = a->C; g.K = a->R;
  g.A = a->v; g.a_rs = a->R; g.a_cs = 1;
  g.B = a->w_e; g.b_rs = 1; g.b_cs = a->R;
  g.C = a->gate; g.c_rs = a->C; g.alpha = 1.f; g.epi = 2; g.bias = a->b_e;
  e = se_gemm(g, st);
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "se_fc fwd (expand): %s", cudaGetErrorString(e));
  return 0;
}

int se_fc_bwd_launch(const yamb_se_fc_grad* a, cudaStream_t st) {
  if (!a) return set_error(YAMB_EINVAL, "null args");
  int rc = se_fc_check(a->N, a->C, a->R);
  if (rc) return rc;
  if (!a->dgate || !a->gate || !a->u || !a->v || !a->pooled || !a->w_r || !a->w_e || !a->dpool ||
      !a->dt || !a->du || !a->g_wr || !a->g_br || !a->g_we || !a->g_be)
    return set_error(YAMB_EINVAL, "se_fc bwd: null pointer");
  // dt = dgate * gate * (1 - gate), db_e += column sums
  {
    const int rows = 32;
    dim3 grid((a->C + 255) / 256, (a->N + rows - 1) / rows);
    se_dt_kernel<<<grid, 256, 0, st>>>(a->N, a->C, a->dgate, a->gate, a->dt, a->g_be, rows);
  }
  SeGemm g;
  cudaError_t e;
  // du[N][R] = (dt[N][C] * W_e[C][R]) * act'(u), db_r += column sums
  memset(&g, 0, sizeof(g));
  g.M = a->N; g.N = a->R; g.K = a->C;
  g.A = a->dt; g.a_rs = a->C; g.a_cs = 1;
  g.B = a->w_e; g.b_rs = a->R; g.b_cs = 1;
  g.C = a->du; g.c_rs = a->R; g.alpha = 1.f; g.epi = 5;
  e = cudaMemsetAsync(a->du, 0, (size_t)a->N * a->R * sizeof(float), st);
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "se_fc memset: %s", cudaGetErrorString(e));
  if ((e = se_gemm(g, st, se_ksplit(g.M, g.N, g.K))) != cudaSuccess)
    return set_error(YAMB_ECUDA, "se_fc bwd (du): %s", cudaGetErrorString(e));
  {
    dim3 fg((a->R + 255) / 256, (a->N + 31) / 32);
    se_finish_kernel<<<fg, 256, 0, st>>>(a->N, a->R, a->du, nullptr, nullptr, a->u, a->g_br, a->act, 1);
  }
  // dpool[N][C] = inv_hw * du[N][R] * W_r[R][C]
  memset(&g, 0, sizeof(g));
  g.M = a->N; g.N = a->C; g.K = a->R;
  g.A = a->du; g.a_rs = a->R; g.a_cs = 1;
  g.B = a->w_r; g.b_rs = a->C; g.b_cs = 1;
  g.C = a->dpool; g.c_rs = a->C; g.alpha = a->inv_hw; g.epi = 0;
  if ((e = se_gemm(g, st)) != cudaSuccess) return set_error(YAMB_ECUDA, "se_fc bwd (dpool): %s", cudaGetErrorString(e));
  // dW_e[C][R] += dt^T[C][N] * v[N][R]
  memset(&g, 0, sizeof(g));
  g.M = a->C; g.N = a->R; g.K = a->N;
  g.A = a->dt; g.a_rs = 1; g.a_cs = a->C;
  g.B = a->v; g.b_rs = a->R; g.b_cs = 1;
  g.C = a->g_we; g.c_rs = a->R; g.alpha = 1.f; g.epi = 4;
  if ((e = se_gemm(g, st)) != cudaSuccess) return set_error(YAMB_ECUDA, "se_fc bwd (dW_e): %s", cudaGetErrorString(e));
  // dW_r[R][C] += du^T[R][N] * s[N][C]
  memset(&g, 0, sizeof(g));
  g.M = a->R; g.N = a->C; g.K = a->N;
  g.A = a->du; g.a_rs = 1; g.a_cs = a->R;
  g.B = a->pooled; g.b_rs = a->C; g.b_cs = 1;
  g.C = a->g_wr; g.c_rs = a->C; g.alpha = 1.f; g.epi = 4;
  if ((e = se_gemm(g, st)) != cudaSuccess) return set_error(YAMB_ECUDA, "se_fc bwd (dW_r): %s", cudaGetErrorString(e));
  return 0;
}

}  // namespace yamb
