// Deterministic reductions.  Kernels whose CTAs (or split-K slabs) all contribute to one output
// write their partial sums with plain stores into a scratch buffer, one slab per producer, and
// det_reduce_launch adds the slabs into the output in slab order.  Float atomics would add them in
// whatever order the CTAs finish, so a training run would not compute the same bits twice.
//
// The scratch of every launch is its own stream-ordered allocation (cudaMallocAsync), released on
// the same stream right after the reduction: launches on different streams never share it, and in
// a CUDA-graph capture it becomes an allocation node owned by the graph, valid whenever the graph
// is replayed.
#include <cuda_runtime.h>

#include <stdint.h>

#include <mutex>

#include "host_util.h"

namespace yamb {

int det_alloc(size_t bytes, cudaStream_t st, float** out) {
  // Keep freed blocks in the device's default pool instead of returning them to the driver at
  // every synchronisation: the same sizes are requested again on the next training step.
  static std::once_flag once[16];
  int dev = 0;
  if (cudaGetDevice(&dev) == cudaSuccess && dev >= 0 && dev < 16) {
    std::call_once(once[dev], [dev] {
      cudaMemPool_t pool;
      if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
        uint64_t keep = UINT64_MAX;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
      }
    });
  }
  void* p = nullptr;
  cudaError_t e = cudaMallocAsync(&p, bytes, st);
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "reduction scratch (%zu bytes): %s", bytes, cudaGetErrorString(e));
  *out = static_cast<float*>(p);
  return 0;
}

int det_free(float* part, cudaStream_t st) {
  cudaError_t e = cudaFreeAsync(part, st);
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "reduction scratch free: %s", cudaGetErrorString(e));
  return 0;
}

// out[i] (+)= sum over s = 0 .. nslab-1 of part[s * n + i], in that order
__global__ void __launch_bounds__(256) det_reduce_kernel(const float* __restrict__ part, int nslab,
                                                         long long n, float* __restrict__ out,
                                                         bool add) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    float s = 0.f;
    for (int k = 0; k < nslab; ++k) s += part[(size_t)k * n + i];
    out[i] = add ? out[i] + s : s;
  }
}

int det_reduce_launch(float* part, int nslab, long long n, float* out, cudaStream_t st, bool add) {
  if (n > 0 && nslab > 0) {
    const long long blocks = (n + 255) / 256;
    const long long cap = 4LL * (max_ctas() > 0 ? max_ctas() : 1);
    det_reduce_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>(part, nslab, n, out, add);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
      det_free(part, st);
      return set_error(YAMB_ECUDA, "det_reduce launch: %s", cudaGetErrorString(e));
    }
  }
  return det_free(part, st);
}

}  // namespace yamb
