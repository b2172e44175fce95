// The depthwise of up to three branches of a multi-branch block in one launch each way
// (yamb_depthwise_fwd_grouped / _bwd_grouped, include/yamb200.h).
//
// Horizontal fusion of the per-branch launches: the grid is the concatenation of the grids the
// per-branch launches use (sized by the same dispatch, grid_k in depthwise.cuh), cut into segments
// — one per branch forward; backward one per branch plus, for k = 7, one for the second
// (taps 25..48) weight-gradient kernel.  CTA j finds its segment from the prefix sums and runs, as
// virtual CTA (j - start, of a grid of the segment's size), the kernel text of the per-branch
// kernel (depthwise_fwd_kernel.cuh / depthwise_bwd_kernel.cuh, included here as device functions):
// the same instantiation, tile range, pointers, weight-gradient slab and statistics slice, so every
// output has the per-branch bits.  A branch's statistics are finalised by the last of its own CTAs
// (arrive_last_of on its own counter).
//
// One kernel per stride holds every instantiation of that stride; a CTA branches once, on its
// segment's key.  Its register count is the largest of them, so the 3x3 segments run at the
// occupancy of the widest kernel (one CTA per SM where the per-branch 3x3 kernels have two).
#include <climits>

#include "depthwise.cuh"

#define YAMB_DW_GROUPED 1
#define YAMB_DW_BWD_SE 0
#define YAMB_DW_BID vbid
#define YAMB_DW_NBLK vnblk
#define YAMB_DW_ARRIVE_LAST(counter) arrive_last_of(counter, vnblk)

namespace yamb {

#include "depthwise_fwd_kernel.cuh"
#include "depthwise_bwd_kernel.cuh"

#undef YAMB_DW_GROUPED
#undef YAMB_DW_BWD_SE
#undef YAMB_DW_BID
#undef YAMB_DW_NBLK
#undef YAMB_DW_ARRIVE_LAST

constexpr int kMaxBr = YAMB_DW_MAX_BRANCHES;
constexpr int kMaxSeg = 2 * kMaxBr;

// instantiation key of a segment: k, channel tile and (forward) tile width or (backward) part
// (0: the dgrad + taps 0..24 kernel, 1: the taps 25..48 kernel of k = 7)
__host__ __device__ constexpr int seg_key(int k, int ct, int x) { return k * 1000 + ct * 10 + x; }

struct DwFwdGroupDev {
  DwFwdDev br[kMaxBr];
  int start[kMaxBr + 1];   // prefix sums of the branch grids
  int key[kMaxBr];
  int nseg;
};

struct DwBwdGroupDev {
  DwBwdDev br[kMaxBr];
  int start[kMaxSeg + 1];
  int branch[kMaxSeg];
  int key[kMaxSeg];
  int nseg;
};

__device__ __forceinline__ int find_seg(const int* start, int nseg) {
  int b = 0;
  while (b + 1 < nseg && (int)blockIdx.x >= start[b + 1]) ++b;
  return b;
}

template <int S>
__global__ void __launch_bounds__(256, 1) dw_fwd_grouped_kernel(
    const __grid_constant__ DwFwdGroupDev g) {
  const int b = find_seg(g.start, g.nseg);
  const unsigned vbid = blockIdx.x - g.start[b], vnblk = g.start[b + 1] - g.start[b];
  const DwFwdDev& p = g.br[b];
  switch (g.key[b]) {
#define YAMB_FWD_SEG(KK, CC, TT) \
    case seg_key(KK, CC, TT): dw_fwd_body<KK, S, CC, TT>(p, vbid, vnblk); break;
#define YAMB_FWD_SEG_CT(CC) \
    YAMB_FWD_SEG(3, CC, 1) YAMB_FWD_SEG(3, CC, 2) YAMB_FWD_SEG(5, CC, 1) YAMB_FWD_SEG(5, CC, 2) \
    YAMB_FWD_SEG(7, CC, 1)
    YAMB_FWD_SEG_CT(8) YAMB_FWD_SEG_CT(16) YAMB_FWD_SEG_CT(32) YAMB_FWD_SEG_CT(64)
#undef YAMB_FWD_SEG_CT
#undef YAMB_FWD_SEG
    default: break;
  }
}

template <int S>
__global__ void __launch_bounds__(256, 1) dw_bwd_grouped_kernel(
    const __grid_constant__ DwBwdGroupDev g) {
  const int sg = find_seg(g.start, g.nseg);
  const unsigned vbid = blockIdx.x - g.start[sg], vnblk = g.start[sg + 1] - g.start[sg];
  const DwBwdDev& p = g.br[g.branch[sg]];
  switch (g.key[sg]) {
#define YAMB_BWD_SEG_CT(CC)                                                                        \
    case seg_key(3, CC, 0): dw_bwd_body<3, S, CC, 0, 9, true>(p, vbid, vnblk); break;              \
    case seg_key(5, CC, 0): dw_bwd_body<5, S, CC, 0, 25, true>(p, vbid, vnblk); break;             \
    case seg_key(7, CC, 0): dw_bwd_body<7, S, CC, 0, 25, true>(p, vbid, vnblk); break;             \
    case seg_key(7, CC, 1): dw_bwd_body<7, S, CC, 25, 49, false>(p, vbid, vnblk); break;
    YAMB_BWD_SEG_CT(8) YAMB_BWD_SEG_CT(16) YAMB_BWD_SEG_CT(32) YAMB_BWD_SEG_CT(64)
#undef YAMB_BWD_SEG_CT
    default: break;
  }
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
// The checks that need no device: count, one stride, distinct statistics counters, each branch's
// own checks (dw_*_setup without the device), and (want_grids) positive grids whose sum fits an int.
template <typename Args>
static int check_group(const Args* a, const char* fn) {
  if (!a) return set_error(YAMB_EINVAL, "%s: null args", fn);
  if (a->nbranch < 1 || a->nbranch > kMaxBr)
    return set_error(YAMB_EINVAL, "%s: nbranch=%d (1..%d)", fn, a->nbranch, kMaxBr);
  for (int b = 0; b < a->nbranch; ++b) {
    if (a->branch[b].stride != a->branch[0].stride)
      return set_error(YAMB_EINVAL, "%s: branches of different strides", fn);
    for (int c = 0; c < b; ++c)
      if (a->branch[b].bn && a->branch[c].bn && a->branch[b].bn->counter == a->branch[c].bn->counter)
        return set_error(YAMB_EINVAL, "%s: branches %d and %d share a statistics counter", fn, c, b);
  }
  return 0;
}

static int check_grids(const int32_t* grid, const int32_t* grid_wgrad, const int* k, int n,
                       const char* fn) {
  long long total = 0;
  for (int b = 0; b < n; ++b) {
    if (grid[b] <= 0) return set_error(YAMB_EINVAL, "%s: grid[%d]=%d", fn, b, grid[b]);
    total += grid[b];
    if (grid_wgrad) {
      if ((k[b] == 7) != (grid_wgrad[b] > 0) || grid_wgrad[b] < 0)
        return set_error(YAMB_EINVAL, "%s: grid_wgrad[%d]=%d with k=%d", fn, b, grid_wgrad[b], k[b]);
      total += grid_wgrad[b];
    }
  }
  if (total > INT_MAX) return set_error(YAMB_EINVAL, "%s: grid too large", fn);
  return 0;
}

struct FwdPlan {
  DwFwdDev p[kMaxBr];
  int ct[kMaxBr], tw[kMaxBr], k[kMaxBr];
  size_t smem[kMaxBr];
};

static int fwd_plan(const yamb_dw_fwd_grouped* a, FwdPlan* pl, const char* fn) {
  int rc = check_group(a, fn);
  for (int b = 0; !rc && b < a->nbranch; ++b) {
    rc = dw_fwd_setup(&a->branch[b], &pl->p[b], &pl->ct[b], &pl->tw[b], &pl->smem[b], false);
    pl->k[b] = a->branch[b].k;
  }
  return rc;
}

struct BwdPlan {
  DwBwdDev p[kMaxBr];
  int ct[kMaxBr], k[kMaxBr];
  size_t smem[kMaxBr];
};

static int bwd_plan(const yamb_dw_bwd_grouped* a, BwdPlan* pl, const char* fn) {
  int rc = check_group(a, fn);
  for (int b = 0; !rc && b < a->nbranch; ++b) {
    rc = dw_bwd_setup(&a->branch[b], &pl->p[b], &pl->ct[b], &pl->smem[b], false);
    pl->k[b] = a->branch[b].k;
  }
  return rc;
}

// grids of the per-branch launches on this device (the same dispatch, in sizing mode)
static int fwd_grids(const FwdPlan& pl, int n, int s, int32_t* grid) {
  for (int b = 0; b < n; ++b) {
    int g = 0;
    int rc = dw_fwd_dispatch(pl.p[b], pl.k[b], s, pl.ct[b], pl.tw[b], pl.smem[b], 0, &g);
    if (rc) return rc;
    grid[b] = g;
  }
  return 0;
}

static int bwd_grids(const BwdPlan& pl, int n, int s, int32_t* grid, int32_t* grid_wgrad) {
  for (int b = 0; b < n; ++b) {
    int g[2] = {0, 0};
    int rc = dw_bwd_dispatch(pl.p[b], pl.k[b], s, pl.ct[b], pl.smem[b], 0, g);
    if (rc) return rc;
    grid[b] = g[0];
    grid_wgrad[b] = g[1];
  }
  return 0;
}

template <typename Kern, typename Dev>
static int launch_group(const char* fn, Kern kern, const Dev& g, int grid, size_t smem,
                        cudaStream_t st) {
  int rc = smem_optin(fn, (const void*)kern, smem);
  if (rc) return rc;
  kern<<<grid, 256, smem, st>>>(g);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(YAMB_ECUDA, "%s: %s", fn, cudaGetErrorString(e));
  return 0;
}

int dw_fwd_grouped_launch(const yamb_dw_fwd_grouped* a, cudaStream_t st) {
  const char* fn = "depthwise fwd grouped";
  FwdPlan pl;
  int rc = fwd_plan(a, &pl, fn);
  if (!rc) rc = check_grids(a->grid, nullptr, pl.k, a->nbranch, fn);
  if (rc) return rc;
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  const int n = a->nbranch, s = a->branch[0].stride;
  int32_t want[kMaxBr];
  if ((rc = fwd_grids(pl, n, s, want))) return rc;
  DwFwdGroupDev g;
  size_t smem = 0;
  g.start[0] = 0;
  for (int b = 0; b < n; ++b) {
    if (a->grid[b] != want[b])
      return set_error(YAMB_EINVAL, "%s: grid[%d]=%d, the branch's own launch uses %d", fn, b,
                       a->grid[b], want[b]);
    g.br[b] = pl.p[b];
    g.key[b] = seg_key(pl.k[b], pl.ct[b], pl.tw[b]);
    g.start[b + 1] = g.start[b] + want[b];
    if (pl.smem[b] > smem) smem = pl.smem[b];
  }
  g.nseg = n;
  return s == 1 ? launch_group(fn, dw_fwd_grouped_kernel<1>, g, g.start[n], smem, st)
                : launch_group(fn, dw_fwd_grouped_kernel<2>, g, g.start[n], smem, st);
}

int dw_bwd_grouped_launch(const yamb_dw_bwd_grouped* a, cudaStream_t st) {
  const char* fn = "depthwise bwd grouped";
  BwdPlan pl;
  int rc = bwd_plan(a, &pl, fn);
  if (!rc) rc = check_grids(a->grid, a->grid_wgrad, pl.k, a->nbranch, fn);
  if (rc) return rc;
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  const int n = a->nbranch, s = a->branch[0].stride;
  int32_t want[kMaxBr], want2[kMaxBr];
  if ((rc = bwd_grids(pl, n, s, want, want2))) return rc;
  DwBwdGroupDev g;
  size_t smem = 0;
  int nseg = 0;
  g.start[0] = 0;
  for (int b = 0; b < n; ++b) {
    if (a->grid[b] != want[b] || a->grid_wgrad[b] != want2[b])
      return set_error(YAMB_EINVAL, "%s: grids of branch %d are %d/%d, its own launch uses %d/%d",
                       fn, b, a->grid[b], a->grid_wgrad[b], want[b], want2[b]);
    g.br[b] = pl.p[b];
    for (int part = 0; part < (want2[b] > 0 ? 2 : 1); ++part) {
      g.branch[nseg] = b;
      g.key[nseg] = seg_key(pl.k[b], pl.ct[b], part);
      g.start[nseg + 1] = g.start[nseg] + (part ? want2[b] : want[b]);
      ++nseg;
    }
    if (pl.smem[b] > smem) smem = pl.smem[b];
  }
  g.nseg = nseg;
  // weight gradient: per-branch slabs (one per CTA of the branch's larger kernel, zero-filled),
  // added in slab order after the kernel, as the per-branch launch does
  int slabs[kMaxBr];
  long long nw[kMaxBr];
  int nalloc = 0;
  cudaError_t e = cudaSuccess;
  for (int b = 0; b < n && !rc; ++b) {
    slabs[b] = want[b] > want2[b] ? want[b] : want2[b];
    nw[b] = (long long)pl.p[b].C * pl.k[b] * pl.k[b];
    const size_t bytes = (size_t)(slabs[b] * nw[b]) * sizeof(float);
    rc = det_alloc(bytes, st, &g.br[b].part);
    if (rc) break;
    ++nalloc;
    e = cudaMemsetAsync(g.br[b].part, 0, bytes, st);
    if (e != cudaSuccess) rc = set_error(YAMB_ECUDA, "%s: %s", fn, cudaGetErrorString(e));
  }
  if (!rc)
    rc = s == 1 ? launch_group(fn, dw_bwd_grouped_kernel<1>, g, g.start[nseg], smem, st)
                : launch_group(fn, dw_bwd_grouped_kernel<2>, g, g.start[nseg], smem, st);
  if (rc) {
    for (int b = 0; b < nalloc; ++b) det_free(g.br[b].part, st);
    return rc;
  }
  for (int b = 0; b < n; ++b) {
    // det_reduce_launch releases the scratch it reduces, also when it fails
    const int r = det_reduce_launch(g.br[b].part, slabs[b], nw[b], pl.p[b].dw, st);
    if (r && !rc) rc = r;
  }
  return rc;
}

int dw_grouped_grids(yamb_dw_fwd_grouped* f, yamb_dw_bwd_grouped* bw) {
  FwdPlan fp;
  BwdPlan bp;
  int rc = 0;
  if (f) rc = fwd_plan(f, &fp, "depthwise fwd grouped");
  if (!rc && bw) rc = bwd_plan(bw, &bp, "depthwise bwd grouped");
  if (rc) return rc;
  if (max_ctas() <= 0) return set_error(YAMB_ENODEV, "no CUDA device");
  if (f) rc = fwd_grids(fp, f->nbranch, f->branch[0].stride, f->grid);
  if (!rc && bw) rc = bwd_grids(bp, bw->nbranch, bw->branch[0].stride, bw->grid, bw->grid_wgrad);
  return rc;
}

}  // namespace yamb
