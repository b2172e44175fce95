// Fused flat-arena optimizer steps, sm_90a.  One launch replaces the ~7 ATen launches per tensor
// of the reference's Python-loop RMSprop (utils/rmsprop.py:67-129), or the per-tensor loop of
// torch.optim.SGD (utils/optim.py:262-267), the L2 penalty's autograd
// graph (utils/optim.py:177-200, folded as grad += wd[i]*p), the DDP mean (utils/distributed.py:136,
// folded as grad_scale = 1/world), the EMA update (utils/optim.py:53-64) and the fp32->bf16 weight
// repack the tensor-core kernels consume.  Pure HBM streaming: float4 accesses, grid-stride.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "host_util.h"
#include "prims.cuh"

namespace yamb {

struct RmsDev {
  long long n;
  float* p; const float* g; float* sq; float* mom; float* grad_avg;
  float* ema; __nv_bfloat16* p_bf16; const unsigned char* wd_mask;
  const float* hyper;  // device [lr, ema_momentum] or NULL
  float lr, alpha, eps, momentum, weight_decay, l2, grad_scale, ema_m;
  int eps_inside_sqrt;
};

// mask byte per element: bit 0 = the 'mnas' L2 term applies, bit 1 = the parameter received no
// gradient this step (reference rmsprop.py:77-78 `if p.grad is None: continue`): only its EMA moves
__device__ __forceinline__ void rms_one(const RmsDev& a, float lr, float ema_m, float& p, float g,
                                        float& sq, float* mom, float* gavg, float* ema,
                                        unsigned mask) {
  const bool l2on = mask & 1u;
  if (mask & 2u) {
    if (ema) *ema = *ema * ema_m + (1.f - ema_m) * p;
    return;
  }
  g *= a.grad_scale;
  if (l2on) g = fmaf(a.l2, p, g);                       // d/dp 0.5*wd*p^2 (optim.py:193-200)
  if (a.weight_decay != 0.f) g = fmaf(a.weight_decay, p, g);  // rmsprop.py:99-100
  sq = sq * a.alpha + (1.f - a.alpha) * g * g;          // rmsprop.py:102
  float avg;
  if (gavg) {                                           // centered, rmsprop.py:104-112
    *gavg = *gavg * a.alpha + (1.f - a.alpha) * g;
    float v = sq - (*gavg) * (*gavg);
    avg = a.eps_inside_sqrt ? sqrtf(v + a.eps) : sqrtf(v) + a.eps;
  } else {
    avg = a.eps_inside_sqrt ? sqrtf(sq + a.eps) : sqrtf(sq) + a.eps;  // :114-117
  }
  if (mom) {                                            // :119-122
    *mom = *mom * a.momentum + g / avg;
    p = p - lr * (*mom);
  } else {
    p = p - lr * (g / avg);                             // :123-124
  }
  if (ema) *ema = *ema * ema_m + (1.f - ema_m) * p;     // optim.py:63-64
}

__global__ void __launch_bounds__(256) rmsprop_kernel(const __grid_constant__ RmsDev a) {
  const float lr = a.hyper ? a.hyper[0] : a.lr;
  const float ema_m = a.hyper ? a.hyper[1] : a.ema_m;
  const long long n4 = a.n / 4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 p = reinterpret_cast<float4*>(a.p)[i];
    const float4 g = reinterpret_cast<const float4*>(a.g)[i];
    float4 sq = reinterpret_cast<float4*>(a.sq)[i];
    float4 mo = a.mom ? reinterpret_cast<float4*>(a.mom)[i] : make_float4(0, 0, 0, 0);
    float4 ga = a.grad_avg ? reinterpret_cast<float4*>(a.grad_avg)[i] : make_float4(0, 0, 0, 0);
    float4 em = a.ema ? reinterpret_cast<float4*>(a.ema)[i] : make_float4(0, 0, 0, 0);
    uchar4 wm = a.wd_mask ? reinterpret_cast<const uchar4*>(a.wd_mask)[i] : make_uchar4(0, 0, 0, 0);
    rms_one(a, lr, ema_m, p.x, g.x, sq.x, a.mom ? &mo.x : nullptr, a.grad_avg ? &ga.x : nullptr,
            a.ema ? &em.x : nullptr, wm.x);
    rms_one(a, lr, ema_m, p.y, g.y, sq.y, a.mom ? &mo.y : nullptr, a.grad_avg ? &ga.y : nullptr,
            a.ema ? &em.y : nullptr, wm.y);
    rms_one(a, lr, ema_m, p.z, g.z, sq.z, a.mom ? &mo.z : nullptr, a.grad_avg ? &ga.z : nullptr,
            a.ema ? &em.z : nullptr, wm.z);
    rms_one(a, lr, ema_m, p.w, g.w, sq.w, a.mom ? &mo.w : nullptr, a.grad_avg ? &ga.w : nullptr,
            a.ema ? &em.w : nullptr, wm.w);
    reinterpret_cast<float4*>(a.p)[i] = p;
    reinterpret_cast<float4*>(a.sq)[i] = sq;
    if (a.mom) reinterpret_cast<float4*>(a.mom)[i] = mo;
    if (a.grad_avg) reinterpret_cast<float4*>(a.grad_avg)[i] = ga;
    if (a.ema) reinterpret_cast<float4*>(a.ema)[i] = em;
    if (a.p_bf16)
      reinterpret_cast<uint2*>(a.p_bf16)[i] = make_uint2(pack_bf16(p.x, p.y), pack_bf16(p.z, p.w));
  }
  // tail (n % 4)
  for (long long i = n4 * 4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n;
       i += (long long)gridDim.x * blockDim.x) {
    float p = a.p[i], sq = a.sq[i];
    float mo = a.mom ? a.mom[i] : 0.f, ga = a.grad_avg ? a.grad_avg[i] : 0.f;
    float em = a.ema ? a.ema[i] : 0.f;
    rms_one(a, lr, ema_m, p, a.g[i], sq, a.mom ? &mo : nullptr, a.grad_avg ? &ga : nullptr,
            a.ema ? &em : nullptr, a.wd_mask ? a.wd_mask[i] : 0u);
    a.p[i] = p; a.sq[i] = sq;
    if (a.mom) a.mom[i] = mo;
    if (a.grad_avg) a.grad_avg[i] = ga;
    if (a.ema) a.ema[i] = em;
    if (a.p_bf16) a.p_bf16[i] = __float2bfloat16_rn(p);
  }
}

struct SgdDev {
  long long n;
  float* p; const float* g; float* mom;
  float* ema; __nv_bfloat16* p_bf16; const unsigned char* wd_mask;
  const float* hyper;  // device [lr, ema_momentum] or NULL
  float lr, momentum, dampening, weight_decay, l2, grad_scale, ema_m;
  int nesterov;
};

// torch.optim.SGD.step (torch/optim/sgd.py, _single_tensor_sgd) for one element.  Mask bits 0 and 1
// as for RMSprop; bit 2 = this parameter takes its first momentum step: torch creates the buffer
// as a copy of the gradient instead of applying the dampened update to a zero buffer
__device__ __forceinline__ void sgd_one(const SgdDev& a, float lr, float ema_m, float& p, float g,
                                        float* mom, float* ema, unsigned mask) {
  if (mask & 2u) {
    if (ema) *ema = *ema * ema_m + (1.f - ema_m) * p;
    return;
  }
  g *= a.grad_scale;
  if (mask & 1u) g = fmaf(a.l2, p, g);                  // d/dp 0.5*wd*p^2 (optim.py:165-176)
  if (a.weight_decay != 0.f) g = fmaf(a.weight_decay, p, g);
  if (mom) {
    const float b = (mask & 4u) ? g : *mom * a.momentum + (1.f - a.dampening) * g;
    *mom = b;
    g = a.nesterov ? fmaf(a.momentum, b, g) : b;
  }
  p = p - lr * g;
  if (ema) *ema = *ema * ema_m + (1.f - ema_m) * p;     // optim.py:63-64
}

__global__ void __launch_bounds__(256) sgd_kernel(const __grid_constant__ SgdDev a) {
  const float lr = a.hyper ? a.hyper[0] : a.lr;
  const float ema_m = a.hyper ? a.hyper[1] : a.ema_m;
  const long long n4 = a.n / 4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 p = reinterpret_cast<float4*>(a.p)[i];
    const float4 g = reinterpret_cast<const float4*>(a.g)[i];
    float4 mo = a.mom ? reinterpret_cast<float4*>(a.mom)[i] : make_float4(0, 0, 0, 0);
    float4 em = a.ema ? reinterpret_cast<float4*>(a.ema)[i] : make_float4(0, 0, 0, 0);
    uchar4 wm = a.wd_mask ? reinterpret_cast<const uchar4*>(a.wd_mask)[i] : make_uchar4(0, 0, 0, 0);
    sgd_one(a, lr, ema_m, p.x, g.x, a.mom ? &mo.x : nullptr, a.ema ? &em.x : nullptr, wm.x);
    sgd_one(a, lr, ema_m, p.y, g.y, a.mom ? &mo.y : nullptr, a.ema ? &em.y : nullptr, wm.y);
    sgd_one(a, lr, ema_m, p.z, g.z, a.mom ? &mo.z : nullptr, a.ema ? &em.z : nullptr, wm.z);
    sgd_one(a, lr, ema_m, p.w, g.w, a.mom ? &mo.w : nullptr, a.ema ? &em.w : nullptr, wm.w);
    reinterpret_cast<float4*>(a.p)[i] = p;
    if (a.mom) reinterpret_cast<float4*>(a.mom)[i] = mo;
    if (a.ema) reinterpret_cast<float4*>(a.ema)[i] = em;
    if (a.p_bf16)
      reinterpret_cast<uint2*>(a.p_bf16)[i] = make_uint2(pack_bf16(p.x, p.y), pack_bf16(p.z, p.w));
  }
  // tail (n % 4)
  for (long long i = n4 * 4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n;
       i += (long long)gridDim.x * blockDim.x) {
    float p = a.p[i];
    float mo = a.mom ? a.mom[i] : 0.f, em = a.ema ? a.ema[i] : 0.f;
    sgd_one(a, lr, ema_m, p, a.g[i], a.mom ? &mo : nullptr, a.ema ? &em : nullptr,
            a.wd_mask ? a.wd_mask[i] : 0u);
    a.p[i] = p;
    if (a.mom) a.mom[i] = mo;
    if (a.ema) a.ema[i] = em;
    if (a.p_bf16) a.p_bf16[i] = __float2bfloat16_rn(p);
  }
}

// shadow <- m*shadow + (1-m)*x  (BN running statistics, utils/optim.py:53-64 / common.py:58-63)
__global__ void ema_kernel(float* shadow, const float* x, long long n, const float* hyper,
                           float m_host) {
  const float m = hyper ? hyper[1] : m_host;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    shadow[i] = shadow[i] * m + (1.f - m) * x[i];
}

__global__ void cast_bf16_kernel(const float* src, __nv_bfloat16* dst, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    dst[i] = __float2bfloat16_rn(src[i]);
}

static int grid_for(long long work) {
  long long b = (work + 255) / 256;
  long long cap = (long long)max_ctas() * 8;
  return (int)(b < 1 ? 1 : (b < cap ? b : cap));
}

int rmsprop_launch(const yamb_rmsprop* a, cudaStream_t st) {
  if (!a || a->n <= 0 || !a->p || !a->g || !a->sq) return set_error(YAMB_EINVAL, "rmsprop args");
  if (a->lr < 0 || a->eps < 0 || a->momentum < 0 || a->weight_decay < 0 || a->alpha < 0)
    return set_error(YAMB_EINVAL, "rmsprop: negative hyper-parameter");  // rmsprop.py:40-50
  if (a->momentum > 0 && !a->mom) return set_error(YAMB_EINVAL, "rmsprop: momentum buffer missing");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  if ((((uintptr_t)a->p) | ((uintptr_t)a->g) | ((uintptr_t)a->sq) | ((uintptr_t)a->mom) |
       ((uintptr_t)a->ema) | ((uintptr_t)a->grad_avg)) & 15)
    return set_error(YAMB_EINVAL, "rmsprop: arenas must be 16-byte aligned");
  RmsDev d;
  d.n = a->n; d.p = a->p; d.g = a->g; d.sq = a->sq;
  d.mom = a->momentum > 0 ? a->mom : nullptr;
  d.grad_avg = a->centered ? a->grad_avg : nullptr;
  d.ema = a->ema; d.p_bf16 = (__nv_bfloat16*)a->p_bf16; d.wd_mask = a->wd_mask;
  d.hyper = a->hyper;
  d.lr = a->lr; d.alpha = a->alpha; d.eps = a->eps; d.momentum = a->momentum;
  d.weight_decay = a->weight_decay; d.l2 = a->l2; d.grad_scale = a->grad_scale; d.ema_m = a->ema_m;
  d.eps_inside_sqrt = a->eps_inside_sqrt;
  rmsprop_kernel<<<grid_for(a->n / 4 + 1), 256, 0, st>>>(d);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "rmsprop: %s", cudaGetErrorString(e));
  return 0;
}

int sgd_launch(const yamb_sgd* a, cudaStream_t st) {
  if (!a || a->n <= 0 || !a->p || !a->g) return set_error(YAMB_EINVAL, "sgd args");
  if (a->lr < 0 || a->momentum < 0 || a->dampening < 0 || a->weight_decay < 0)
    return set_error(YAMB_EINVAL, "sgd: negative hyper-parameter");
  if (a->nesterov && (a->momentum <= 0 || a->dampening != 0))
    return set_error(YAMB_EINVAL, "sgd: nesterov needs momentum > 0 and zero dampening");
  if (a->momentum > 0 && !a->mom) return set_error(YAMB_EINVAL, "sgd: momentum buffer missing");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  if ((((uintptr_t)a->p) | ((uintptr_t)a->g) | ((uintptr_t)a->mom) | ((uintptr_t)a->ema)) & 15)
    return set_error(YAMB_EINVAL, "sgd: arenas must be 16-byte aligned");
  SgdDev d;
  d.n = a->n; d.p = a->p; d.g = a->g;
  d.mom = a->momentum > 0 ? a->mom : nullptr;
  d.ema = a->ema; d.p_bf16 = (__nv_bfloat16*)a->p_bf16; d.wd_mask = a->wd_mask;
  d.hyper = a->hyper;
  d.lr = a->lr; d.momentum = a->momentum; d.dampening = a->dampening;
  d.weight_decay = a->weight_decay; d.l2 = a->l2; d.grad_scale = a->grad_scale; d.ema_m = a->ema_m;
  d.nesterov = a->nesterov;
  sgd_kernel<<<grid_for(a->n / 4 + 1), 256, 0, st>>>(d);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "sgd: %s", cudaGetErrorString(e));
  return 0;
}

int ema_launch(float* shadow, const float* x, long long n, const float* hyper, float m,
               cudaStream_t st) {
  if (!shadow || !x || n <= 0) return set_error(YAMB_EINVAL, "ema args");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  ema_kernel<<<grid_for(n), 256, 0, st>>>(shadow, x, n, hyper, m);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "ema: %s", cudaGetErrorString(e));
  return 0;
}

int cast_bf16_launch(const float* src, void* dst, long long n, cudaStream_t st) {
  if (!src || !dst || n <= 0) return set_error(YAMB_EINVAL, "cast args");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  cast_bf16_kernel<<<grid_for(n), 256, 0, st>>>(src, (__nv_bfloat16*)dst, n);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "cast: %s", cudaGetErrorString(e));
  return 0;
}

}  // namespace yamb
