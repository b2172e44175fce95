// sm_90a device primitives: mbarrier, cp.async, shared-memory vectors, TMA (cp.async.bulk.tensor),
// wgmma.
// Everything here is inline PTX; no CUTLASS dependency.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace yamb {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ----------------------------------------------------------------------------------------------
// thread-block clusters: rank, barrier, distributed shared memory
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// every thread of every CTA of the cluster; orders this CTA's shared-memory writes before the
// peers' reads that follow their wait
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// the address of this CTA's shared-memory word `addr` in the CTA of cluster rank `rank`
__device__ __forceinline__ uint32_t dsmem_map(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ float2 dsmem_ld_f2(uint32_t cluster_addr) {
  float2 v;
  asm volatile("ld.shared::cluster.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(cluster_addr) : "memory");
  return v;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
// try_wait with a suspend-time hint: the hardware parks the thread (no issue slots consumed) until
// the phase completes or ~the hint (ns) elapses.  Without the hint the instruction returns almost
// immediately and a dozen polling warps steal most of the SM's issue bandwidth from the warps
// that do the work (measured: the operand-transform warps ran 4x slower).
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
// Bounded wait: a pipeline bug traps after ~4 s instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  uint64_t t0 = global_timer_ns();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (((++spins) & 0x3fff) == 0) {
      if (global_timer_ns() - t0 > 4000000000ull) {
        printf("yamb: mbarrier timeout block %d thread %d bar %u parity %u\n", (int)blockIdx.x,
               (int)threadIdx.x, smem_u32(bar), parity);
        __trap();
      }
    }
  }
}

// ----------------------------------------------------------------------------------------------
// cp.async (16-byte, L2 only) and 128-bit shared-memory accesses (32-bit shared addresses, never
// generic)
// ----------------------------------------------------------------------------------------------
// copies src_bytes (16 or 0) from src and zero-fills the rest of the 16 bytes at dst: a copy with
// src_bytes = 0 reads nothing, so src need only be a valid address
__device__ __forceinline__ void cp_async_zfill16(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// waits until at most N of this thread's committed groups are still in flight
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t a) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ float4 lds128f(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t a, uint4 v) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w) : "memory");
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* smem_dst,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0),
        "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* m, uint64_t* bar, uint32_t smem_dst,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      :
      : "r"(smem_dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0,
                                             int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               :
               : "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma (sm_90a): D[registers] (+)= A[smem desc] * B[smem desc], issued by a whole warpgroup
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the compiler from moving accumulator reads / writes across a wgmma fence or wait.
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int R, int C>
__device__ __forceinline__ void reg_fence(float (&d)[R][C]) {
#pragma unroll
  for (int i = 0; i < R; ++i) reg_fence(d[i]);
}
// m64nNk16, bf16 x bf16 -> fp32.  TA / TB: 1 = the operand is MN-major in shared memory.
// Accumulator fragment of thread t of the warpgroup (warp w = t / 32, lane l):
//   d[4j + 2h + e]  ->  row 16w + l/4 + 8h,  column 8j + 2(l%4) + e
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
}

// ----------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor (sm_90 format), SWIZZLE_128B, 16-byte units.
//   K-major  tile (rows = M/N, 128B of K per row): LBO unused (1), SBO = 1024B (8 rows x 128B)
//   MN-major tile (rows = K, 128B of M/N per row): LBO = bytes between 64-element MN chunks,
//                                                   SBO = 1024B (8 K-rows x 128B)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t gmma_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes,
                                                   uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3fff);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3fff) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3fff) << 32;
  d |= (uint64_t)1 << 62;  // SWIZZLE_128B
  return d;
}

// ----------------------------------------------------------------------------------------------
// small math helpers
// ----------------------------------------------------------------------------------------------
enum Act : int { ACT_NONE = 0, ACT_RELU = 1, ACT_RELU6 = 2, ACT_SWISH = 3, ACT_HSWISH = 4 };

// swish = z * sigmoid(z): MUFU.EX2 + MUFU.RCP (`__fdividef`, 2 ulp) instead of the IEEE division's
// ~8-instruction sequence — the values are rounded to bf16 (2^-9) right after; exp(-z) = inf gives
// z / inf = -0, the limit.  The operand transforms of the Swish networks are bound by exactly these
// instructions.
__device__ __forceinline__ float act_fwd(float z, int act) {
  switch (act) {
    case ACT_RELU: return fmaxf(z, 0.f);
    case ACT_RELU6: return fminf(fmaxf(z, 0.f), 6.f);
    case ACT_SWISH: return __fdividef(z, 1.f + __expf(-z));
    case ACT_HSWISH: return z * fminf(fmaxf(z + 3.f, 0.f), 6.f) * (1.f / 6.f);
    default: return z;
  }
}
// d act(z) / dz
__device__ __forceinline__ float act_bwd(float z, int act) {
  switch (act) {
    case ACT_RELU: return z > 0.f ? 1.f : 0.f;
    case ACT_RELU6: return (z > 0.f && z < 6.f) ? 1.f : 0.f;
    case ACT_SWISH: {
      float s = __fdividef(1.f, 1.f + __expf(-z));
      return s * (1.f + z * (1.f - s));
    }
    case ACT_HSWISH: return z <= -3.f ? 0.f : (z >= 3.f ? 1.f : (2.f * z + 3.f) * (1.f / 6.f));
    default: return 1.f;
  }
}
// Activation as data: relu / relu6 / none are clamp(z, lo, hi) — two instructions, no branch;
// swish / h-swish take a (warp-uniform) slow branch.
struct ActParam {
  float lo, hi;
  int kind;  // 0: clamp only, else ACT_SWISH / ACT_HSWISH
};
__device__ __forceinline__ ActParam make_act(int act) {
  ActParam a;
  a.lo = (act == ACT_RELU || act == ACT_RELU6) ? 0.f : -3.0e38f;
  a.hi = (act == ACT_RELU6) ? 6.f : 3.0e38f;
  a.kind = (act == ACT_SWISH || act == ACT_HSWISH) ? act : 0;
  return a;
}
__device__ __forceinline__ float act_rt(float z, const ActParam& a) {
  if (a.kind == 0) return fminf(fmaxf(z, a.lo), a.hi);
  if (a.kind == ACT_SWISH) return __fdividef(z, 1.f + __expf(-z));
  return z * fminf(fmaxf(z + 3.f, 0.f), 6.f) * (1.f / 6.f);
}
// d act / dz for the clamp family: 1 strictly inside (lo, hi), else 0
__device__ __forceinline__ float act_bwd_rt(float z, const ActParam& a, int act) {
  if (a.kind == 0) return (z > a.lo && z < a.hi) ? 1.f : 0.f;
  return act_bwd(z, act);
}
// fp32 pair FMA: d = a * b + c on both halves
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

// N-element forms: ONE warp-uniform branch for the whole vector (a branch per element serialises
// the elements: measured 4x slowdown of the operand transform).
template <int N>
__device__ __forceinline__ void act_vec(float (&x)[N], const ActParam& a) {
  if (a.kind == 0) {
#pragma unroll
    for (int i = 0; i < N; ++i) x[i] = fminf(fmaxf(x[i], a.lo), a.hi);
  } else if (a.kind == ACT_SWISH) {
#pragma unroll
    for (int i = 0; i < N; ++i) x[i] = __fdividef(x[i], 1.f + __expf(-x[i]));
  } else {
#pragma unroll
    for (int i = 0; i < N; ++i) x[i] = x[i] * fminf(fmaxf(x[i] + 3.f, 0.f), 6.f) * (1.f / 6.f);
  }
}
// g[i] *= act'(z[i])
template <int N>
__device__ __forceinline__ void act_bwd_vec(float (&g)[N], const float (&z)[N], const ActParam& a,
                                            int act) {
  if (a.kind == 0) {
#pragma unroll
    for (int i = 0; i < N; ++i) g[i] = (z[i] > a.lo && z[i] < a.hi) ? g[i] : 0.f;
  } else {
#pragma unroll
    for (int i = 0; i < N; ++i) g[i] *= act_bwd(z[i], act);
  }
}
__device__ __forceinline__ float bf16lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
// clamp both halves of a bf16x2 word (relu / relu6 after rounding == rounding after the clamp:
// the bounds are bf16 values and rounding is monotonic)
__device__ __forceinline__ uint32_t clamp_bf16x2(uint32_t v, uint32_t lo2, uint32_t hi2) {
  uint32_t d;
  asm("{\n\t.reg .b32 t;\n\tmax.bf16x2 t, %1, %2;\n\tmin.bf16x2 %0, t, %3;\n\t}"
      : "=r"(d)
      : "r"(v), "r"(lo2), "r"(hi2));
  return d;
}
__device__ __forceinline__ float round_bf16(float x) {
  return __bfloat162float(__float2bfloat16_rn(x));
}

}  // namespace yamb
