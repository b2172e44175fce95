// Multi-branch eval block (block_eval_mb.cu, block_eval_mb_cluster.cu): the packed geometry and the
// argument checks and group setup the unsplit and the cluster launchers share.
#pragma once
#include "block_eval.cuh"

namespace yamb {

template <int K_, int S_, int TOH_, int TOW_, int TI_, int CPT_>
struct EvGeomMB : EvGeom<K_, S_, TOH_, TOW_, TI_, CPT_> {
  static constexpr bool MB = true;
};

// kmax in {5, 7}, the expansion, and 1 to 3 groups of strictly decreasing k from channel 0
static int block_eval_mb_check(const yamb_block_eval_mb* m) {
  const yamb_block_eval* a = &m->base;
  if (a->kernel != 5 && a->kernel != 7)
    return set_error(YAMB_EINVAL, "block_eval_mb: kmax in {5,7} (got %d)", a->kernel);
  if (!a->w_expand) return set_error(YAMB_EINVAL, "block_eval_mb: built with expansion only");
  if (m->ngroups < 1 || m->ngroups > 3 || m->group_k[0] != a->kernel || m->group_c0[0] != 0)
    return set_error(YAMB_EINVAL, "block_eval_mb: 1 to 3 groups, the first of k = kmax from channel 0");
  for (int i = 1; i < m->ngroups; ++i)
    if ((m->group_k[i] != 3 && m->group_k[i] != 5) || m->group_k[i] >= m->group_k[i - 1] ||
        m->group_c0[i] <= m->group_c0[i - 1] || m->group_c0[i] % 8 || m->group_c0[i] >= a->Chid)
      return set_error(YAMB_EINVAL, "block_eval_mb: group %d: k decreasing, c0 increasing multiples of 8 < Chid", i);
  return 0;
}

static void block_eval_mb_groups(const yamb_block_eval_mb* m, BlockEvalDev& p) {
  p.ngroups = m->ngroups;
  for (int i = 0; i < 3; ++i) {
    p.gk[i] = i < m->ngroups ? m->group_k[i] : 0;
    p.gc0[i] = i < m->ngroups ? m->group_c0[i] : 0;
  }
}

}  // namespace yamb
