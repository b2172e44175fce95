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
// No float atomics: the split-K products u and du store one slab per K slab and the finish kernel
// adds the slabs in slab order; the bias gradients are column sums per sample slab, added into
// g_b* in slab order by det_reduce.  Every call computes the same bits.
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
  int epi;                           // 0 store alpha*acc | 1 C=sigmoid(acc+bias) | 2 C += acc
                                     // 3 split-K: slab z = blockIdx.z of C, C[z*M*c_rs + m*c_rs + n] = acc
                                     //   (plain stores; the caller adds the slabs in slab order)
  int k_per_slab;                    // K range of one grid.z slab (se_split), 0 = all of K
  const float* bias;                 // [N]
};

constexpr int kSgT = 64, kSgK = 16;

__global__ void __launch_bounds__(256) se_gemm_kernel(const __grid_constant__ SeGemm p) {
  __shared__ float sA[kSgK][kSgT + 4];
  __shared__ float sB[kSgK][kSgT + 4];
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
  float* C = p.epi == 3 ? p.C + (size_t)blockIdx.z * p.M * p.c_rs : p.C;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + tm + i;
    if (m >= p.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tn + j;
      if (n >= p.N) continue;
      float v = acc[i][j] * p.alpha;
      float* c = C + (size_t)m * p.c_rs + n;
      switch (p.epi) {
        case 1: { v += p.bias[n]; *c = 1.f / (1.f + __expf(-v)); break; }
        case 2: *c += v; break;
        default: *c = v;
      }
    }
  }
}

// Sets the K range of one slab for `ksplit` slabs (a multiple of the K chunk) and returns the
// number of slabs the launch writes, which can be less than ksplit.
static int se_split(SeGemm& g, int ksplit) {
  g.k_per_slab = ((g.K + ksplit - 1) / ksplit + kSgK - 1) / kSgK * kSgK;
  return (g.K + g.k_per_slab - 1) / g.k_per_slab;
}

static cudaError_t se_gemm(SeGemm g, cudaStream_t st) {
  if (g.k_per_slab <= 0) g.k_per_slab = g.K;
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

// finish of the split-K products u, du [N][R]; CTA = 32 columns x 8 samples, thread = one
// element: acc = the nslab slabs part[z][N][R] added in slab order, then
//   mode 0: u = acc + b_r, v = act(u)
//   mode 1: du = acc * act'(u_saved), and colpart[blockIdx.y][j] = sum of du over the CTA's 8
//           samples in sample order (one slab of the db_r column sums)
// part may be u (mode 0) or du (mode 1) itself when nslab == 1.
__global__ void __launch_bounds__(256) se_finish_kernel(int N, int R, const float* part, int nslab,
                                                        float* u, float* v, const float* b_r,
                                                        const float* u_saved, float* colpart,
                                                        int act, int mode) {
  __shared__ float s_col[8][33];
  const int j = blockIdx.x * 32 + threadIdx.x, n = blockIdx.y * 8 + threadIdx.y;
  float d = 0.f;
  if (j < R && n < N) {
    const size_t i = (size_t)n * R + j, slab = (size_t)N * R;
    float a = 0.f;
#pragma unroll 4
    for (int z = 0; z < nslab; ++z) a += part[z * slab + i];
    if (mode == 0) {
      const float x = a + b_r[j];
      u[i] = x;
      v[i] = act_fwd(x, act);
    } else {
      d = a * act_bwd(u_saved[i], act);   // here `u` is du
      u[i] = d;
    }
  }
  if (mode == 1) {
    s_col[threadIdx.y][threadIdx.x] = d;
    __syncthreads();
    if (threadIdx.y == 0 && j < R) {
      float s = 0.f;
      for (int r = 0; r < 8; ++r) s += s_col[r][threadIdx.x];
      colpart[(size_t)blockIdx.y * R + j] = s;
    }
  }
}

// dt = dgate * gate * (1 - gate); colpart[blockIdx.y][c] = sum of dt over this CTA's samples (one
// slab of the db_e column sums)          thread = channel, CTA = sample slab
__global__ void __launch_bounds__(256) se_dt_kernel(int N, int C, const float* dgate, const float* gate,
                                                    float* dt, float* colpart, int rows_per_cta) {
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
  colpart[(size_t)blockIdx.y * C + c] = s;
}

static int se_fc_check(int N, int C, int R) {
  if (N <= 0 || C <= 0 || R <= 0 || C > 4096 || R > 1024 || N > 8 * 65535)
    return set_error(YAMB_EINVAL, "se_fc: N=%d C=%d R=%d", N, C, R);
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  return 0;
}

// The split-K product [N][R] (u or du) of g, K = C: each K slab stored into its own slab of a
// stream-ordered scratch *part, or straight into `out` when there is only one slab (*part = out).
// The slab count depends on the shape and the device only, so the order of the sum does too.
static int se_split_product(SeGemm g, float* out, cudaStream_t st, float** part, int* nslab,
                            const char* what) {
  *nslab = se_split(g, se_ksplit(g.M, g.N, g.K));
  *part = out;
  if (*nslab > 1) {
    int rc = det_alloc((size_t)*nslab * g.M * g.N * sizeof(float), st, part);
    if (rc) return rc;
  }
  g.C = *part; g.c_rs = g.N; g.epi = 3;
  cudaError_t e = se_gemm(g, st);
  if (e != cudaSuccess) {
    if (*part != out) det_free(*part, st);
    return set_error(YAMB_ECUDA, "se_fc %s: %s", what, cudaGetErrorString(e));
  }
  return 0;
}

// se_finish_kernel launch check; releases the split-K scratch
static int se_finish_done(float* part, float* out, cudaStream_t st, const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    if (part != out) det_free(part, st);
    return set_error(YAMB_ECUDA, "se_fc %s: %s", what, cudaGetErrorString(e));
  }
  return part != out ? det_free(part, st) : 0;
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
  g.alpha = 1.f;
  float* part;
  int nslab;
  if ((rc = se_split_product(g, a->u, st, &part, &nslab, "fwd (reduce)"))) return rc;
  {
    dim3 fg((a->R + 31) / 32, (a->N + 7) / 8);
    se_finish_kernel<<<fg, dim3(32, 8), 0, st>>>(a->N, a->R, part, nslab, a->u, a->v, a->b_r,
                                                 nullptr, nullptr, a->act, 0);
    if ((rc = se_finish_done(part, a->u, st, "fwd (finish)"))) return rc;
  }
  // gate[N][C] = sigmoid(v[N][R] * W_e[C][R]^T + b_e)
  memset(&g, 0, sizeof(g));
  g.M = a->N; g.N = a->C; g.K = a->R;
  g.A = a->v; g.a_rs = a->R; g.a_cs = 1;
  g.B = a->w_e; g.b_rs = 1; g.b_cs = a->R;
  g.C = a->gate; g.c_rs = a->C; g.alpha = 1.f; g.epi = 1; g.bias = a->b_e;
  cudaError_t e = se_gemm(g, st);
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
  cudaError_t e;
  float* colpart;
  // dt = dgate * gate * (1 - gate), db_e += column sums (slabs of 32 samples)
  int nrow = (a->N + 31) / 32;
  if ((rc = det_alloc((size_t)nrow * a->C * sizeof(float), st, &colpart))) return rc;
  {
    dim3 grid((a->C + 255) / 256, nrow);
    se_dt_kernel<<<grid, 256, 0, st>>>(a->N, a->C, a->dgate, a->gate, a->dt, colpart, 32);
    if ((e = cudaGetLastError()) != cudaSuccess) {
      det_free(colpart, st);
      return set_error(YAMB_ECUDA, "se_fc bwd (dt): %s", cudaGetErrorString(e));
    }
  }
  if ((rc = det_reduce_launch(colpart, nrow, a->C, a->g_be, st))) return rc;
  SeGemm g;
  // du[N][R] = (dt[N][C] * W_e[C][R]) * act'(u), db_r += column sums (slabs of 8 samples)
  memset(&g, 0, sizeof(g));
  g.M = a->N; g.N = a->R; g.K = a->C;
  g.A = a->dt; g.a_rs = a->C; g.a_cs = 1;
  g.B = a->w_e; g.b_rs = a->R; g.b_cs = 1;
  g.alpha = 1.f;
  float* part;
  int nslab;
  nrow = (a->N + 7) / 8;
  if ((rc = det_alloc((size_t)nrow * a->R * sizeof(float), st, &colpart))) return rc;
  if ((rc = se_split_product(g, a->du, st, &part, &nslab, "bwd (du)"))) {
    det_free(colpart, st);
    return rc;
  }
  {
    dim3 fg((a->R + 31) / 32, nrow);
    se_finish_kernel<<<fg, dim3(32, 8), 0, st>>>(a->N, a->R, part, nslab, a->du, nullptr, nullptr,
                                                 a->u, colpart, a->act, 1);
    if ((rc = se_finish_done(part, a->du, st, "bwd (du finish)"))) {
      det_free(colpart, st);
      return rc;
    }
  }
  if ((rc = det_reduce_launch(colpart, nrow, a->R, a->g_br, st))) return rc;
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
  g.C = a->g_we; g.c_rs = a->R; g.alpha = 1.f; g.epi = 2;
  if ((e = se_gemm(g, st)) != cudaSuccess) return set_error(YAMB_ECUDA, "se_fc bwd (dW_e): %s", cudaGetErrorString(e));
  // dW_r[R][C] += du^T[R][N] * s[N][C]
  memset(&g, 0, sizeof(g));
  g.M = a->R; g.N = a->C; g.K = a->N;
  g.A = a->du; g.a_rs = 1; g.a_cs = a->R;
  g.B = a->pooled; g.b_rs = a->C; g.b_cs = 1;
  g.C = a->g_wr; g.c_rs = a->C; g.alpha = 1.f; g.epi = 2;
  if ((e = se_gemm(g, st)) != cudaSuccess) return set_error(YAMB_ECUDA, "se_fc bwd (dW_r): %s", cudaGetErrorString(e));
  return 0;
}

}  // namespace yamb
