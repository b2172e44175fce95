// Eval-mode multi-branch inverted-residual block (several depthwise kernel sizes: AtomNAS) in one
// launch, plus the packing kernel that lays its branches out as one hidden dimension.
//
// The branches' hidden channels are packed into groups of decreasing k (7, 5, 3), each branch padded
// to a multiple of 8 channels; the block kernel of block_eval.cuh then runs over the packed block
// with the tile of K_MAX and, per 64-channel slice, the stencil of the slice's own k (EvGeomMB: the
// G::MB branches of the kernel body).  The tap table is zero-embedded in the centre of
// K_MAX x K_MAX, so a boundary slice that runs the larger stencil over a few smaller-k channels adds
// products with zero taps, and the centred window of a smaller-k slice is the same convolution as
// the branch's own (padding (k - 1) / 2 for every k).  Padded channels have zero W1 rows and W3
// columns and BatchNorms that map 0 to 0: they contribute nothing.
#include "block_eval_mb.cuh"

namespace yamb {

// ---- packing: one CTA per packed hidden channel ---------------------------------------------------
struct MbPackDev {
  yamb_block_eval_mb_pack_args a;
};

__global__ void __launch_bounds__(128) block_eval_mb_pack_kernel(const __grid_constant__ MbPackDev d) {
  const yamb_block_eval_mb_pack_args& a = d.a;
  const int j = blockIdx.x, tid = threadIdx.x;
  const int code = __ldg(a.map + j);
  const bool pad = code < 0;
  const yamb_mb_branch& b = a.branch[pad ? 0 : (code >> 16)];
  const int c = pad ? 0 : (code & 0xffff);
  const int K = a.kmax, k = b.k, off = (K - k) / 2;
  __nv_bfloat16* w1 = reinterpret_cast<__nv_bfloat16*>(a.w_expand);
  __nv_bfloat16* w3 = reinterpret_cast<__nv_bfloat16*>(a.w_project);
  for (int i = tid; i < a.Cin; i += 128)
    w1[(size_t)j * a.Cin + i] = __float2bfloat16_rn(pad ? 0.f : __ldg(b.w_expand + (size_t)c * a.Cin + i));
  for (int i = tid; i < a.Cout; i += 128)
    w3[(size_t)i * a.Chid + j] = __float2bfloat16_rn(pad ? 0.f : __ldg(b.w_project + (size_t)i * b.ld + c));
  for (int i = tid; i < K * K; i += 128) {
    const int ky = i / K - off, kx = i % K - off;
    const bool in = !pad && (unsigned)ky < (unsigned)k && (unsigned)kx < (unsigned)k;
    a.w_dw[(size_t)j * K * K + i] = in ? __ldg(b.w_dw + (size_t)c * k * k + ky * k + kx) : 0.f;
  }
  if (tid < 8) {
    const yamb_bn_eval& bn = tid < 4 ? b.bn1 : b.bn2;
    const int f = tid & 3;
    float v;
    if (pad) v = f == 3 ? 1.f : 0.f;
    else if (f == 0) v = bn.gamma ? __ldg(bn.gamma + c) : 1.f;
    else if (f == 1) v = bn.beta ? __ldg(bn.beta + c) : 0.f;
    else v = __ldg((f == 2 ? bn.running_mean : bn.running_var) + c);
    (tid < 4 ? a.bn1 : a.bn2)[(size_t)f * a.Chid + j] = v;
  }
  if (a.R > 0) {
    for (int r = tid; r < a.R; r += 128) {
      a.se_reduce[(size_t)r * a.Chid + j] = pad ? 0.f : __ldg(b.se_reduce + (size_t)r * b.ld + c);
      a.se_expand[(size_t)j * a.R + r] = pad ? 0.f : __ldg(b.se_expand + (size_t)c * a.R + r);
    }
    if (tid == 0) a.se_expand_bias[j] = pad ? 0.f : __ldg(b.se_expand_bias + c);
  }
}

int block_eval_mb_pack_launch(const yamb_block_eval_mb_pack_args* a, cudaStream_t st) {
  if (!a) return set_error(YAMB_EINVAL, "null args");
  if (a->Cin <= 0 || a->Cout <= 0 || a->Chid <= 0 || a->Chid % 8 || a->R < 0)
    return set_error(YAMB_EINVAL, "block_eval_mb_pack: bad sizes");
  if (a->kmax != 3 && a->kmax != 5 && a->kmax != 7)
    return set_error(YAMB_EINVAL, "block_eval_mb_pack: kmax in {3,5,7} (got %d)", a->kmax);
  if (a->nbranch < 1 || a->nbranch > 3)
    return set_error(YAMB_EINVAL, "block_eval_mb_pack: 1 to 3 branches (got %d)", a->nbranch);
  int total = 0;
  for (int i = 0; i < a->nbranch; ++i) {
    const yamb_mb_branch& b = a->branch[i];
    if ((b.k != 3 && b.k != 5 && b.k != 7) || b.k > a->kmax || b.C <= 0 || b.C > 0xffff)
      return set_error(YAMB_EINVAL, "block_eval_mb_pack: branch %d: k in {3,5,7} <= kmax, 0 < C", i);
    if (!b.w_expand || !b.w_dw || !b.w_project || !b.bn1.running_mean || !b.bn1.running_var ||
        !b.bn2.running_mean || !b.bn2.running_var || (a->R > 0 && (!b.se_reduce || !b.se_expand ||
                                                                 !b.se_expand_bias)))
      return set_error(YAMB_EINVAL, "block_eval_mb_pack: branch %d: null pointer", i);
    if (b.ld < b.C) return set_error(YAMB_EINVAL, "block_eval_mb_pack: ld < branch width");
    total += (b.C + 7) / 8 * 8;
  }
  if (total != a->Chid)
    return set_error(YAMB_EINVAL, "block_eval_mb_pack: Chid %d is not the padded branch total %d",
                     a->Chid, total);
  if (!a->map || !a->w_expand || !a->w_project || !a->w_dw || !a->bn1 || !a->bn2 ||
      (a->R > 0 && (!a->se_reduce || !a->se_expand || !a->se_expand_bias)))
    return set_error(YAMB_EINVAL, "block_eval_mb_pack: null pointer");
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  MbPackDev d;
  d.a = *a;
  block_eval_mb_pack_kernel<<<a->Chid, 128, 0, st>>>(d);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "block_eval_mb_pack launch: %s", cudaGetErrorString(e));
  return 0;
}

// ---- the block ---------------------------------------------------------------------------------
int block_eval_mb_launch(const yamb_block_eval_mb* m, bool pool, cudaStream_t st) {
  if (!m) return set_error(YAMB_EINVAL, "null args");
  const yamb_block_eval* a = &m->base;
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  int rc = block_eval_mb_check(m);
  if (rc) return rc;
  BlockEvalDev p;
  if ((rc = block_eval_setup(a, pool, 1, p))) return rc;
  block_eval_mb_groups(m, p);
  // the tile plan of block_eval_launch_impl for (kmax, stride)
  const bool wide = p.Npad > 16 * kMaxProjChunks;
  auto tiles_of = [&](int toh, int tow, int ti) {
    return (long long)((p.Ho + toh - 1) / toh) * ((p.Wo + tow - 1) / tow) * ((a->N + ti - 1) / ti);
  };
  if (a->kernel == 5) {
    if (a->stride == 2) return launch_eval<EvGeomMB<5, 2, 6, 7, 1, 2>, true, false>(p, a, st);
    if (wide) return launch_eval<EvGeomMB<5, 1, 7, 7, 1, 4>, true, false>(p, a, st);
    if (tiles_of(7, 16, 1) <= tiles_of(7, 7, 2))
      return launch_eval<EvGeomMB<5, 1, 7, 16, 1, 4>, true, false>(p, a, st);
    return launch_eval<EvGeomMB<5, 1, 7, 7, 2, 4>, true, false>(p, a, st);
  }
  if (a->stride == 2) return launch_eval<EvGeomMB<7, 2, 4, 7, 1, 2>, true, false>(p, a, st);
  return launch_eval<EvGeomMB<7, 1, 7, 7, 1, 2>, true, false>(p, a, st);
}

}  // namespace yamb
