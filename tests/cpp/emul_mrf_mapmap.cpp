// tests/cpp/emul_mrf_mapmap.cpp -- fiber emulation (cuda_fiber.h) of one multilevel step of the spanning phase of csrc/mrf.cu,
// as enqueue_multilevel_step drives it after the contraction: k_build_adj4 on the contracted MRF, k_forest<true>,
// k_tree_prep<true>, k_tree<G, 3, true, true> (fast path and the global-memory recursion), the projection, k_energy on the
// faces, k_accept, k_restore of the coarse labels, k_step_count and, for a rejected step, the projection again.  The
// contracted MRF comes from the caller (the contraction kernels are checked against the oracle by
// tests/test_emul_mrf_multilevel.py); the projection is k_ml_project's rule, restated here.  mrf_kernels.inc is the same cut
// of mrf.cu that tests/test_cuda_emulation.py makes.
#include "cuda_fiber.h"

#include <algorithm>
#include <vector>

namespace b2 {
namespace {
alignas(16) unsigned char tree_dyn[256 * 1024];   // k_tree's dynamic shared memory
inline unsigned long long global_timer_ns() { return 0; }
inline void st_release_sys(uint32_t *p, uint32_t v) { *(volatile uint32_t *)p = v; }
inline uint32_t ld_acquire_sys(const uint32_t *p) { return *(const volatile uint32_t *)p; }
}  // namespace
}  // namespace b2

#include "mrf_kernels.inc"

using namespace b2;

namespace {
uint32_t label_pos(const uint64_t *ptr, const uint16_t *view, uint32_t v, uint32_t lab)
{
    uint32_t k = 0;
    while (ptr[v] + k < ptr[v + 1] && (uint32_t)view[ptr[v] + k] + 1u != lab) ++k;
    return ptr[v + 1] > ptr[v] ? k : 0u;
}
// k_ml_project: labels[f] = coarse label of f's node, lidx[f] = its position in f's list
void project(uint32_t F, const uint32_t *region, const uint32_t *clabels, const uint64_t *ptr, const uint16_t *view,
             uint32_t *labels, uint32_t *lidx)
{
    for (uint32_t f = 0; f < F; ++f) {
        labels[f] = clabels[region[f]];
        lidx[f] = label_pos(ptr, view, f, labels[f]);
    }
}
}  // namespace

extern "C" {

// Fine MRF: F, adj_ptr, adj_idx, ptr, view, cost, labels (in: at the start of the step, out: after it).  Contracted MRF: n,
// region [F], cadj_ptr, cadj_idx, cwgt, cptr, cview, ccost, clabels [n] (in: the contracted labels, out: after the step).
// params: [root_div, seed, iteration (>= 1), group (4 / 8 / 16 / 32), longest list the k_tree scratch holds (< 16: the
// longest list of the contracted input)].  level, parent, swept: [n] out (coarse forest, coarse labels after the DP);
// projected: [F] out, the face labels after the DP.  rejected: out, k_accept's decision.
// Returns 0, -1 when a launch hung, -2 on bad parameters, -3 when the counters or energies are inconsistent.
int emul_multilevel_step(uint32_t F, uint32_t K, const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint64_t *ptr,
                         const uint16_t *view, const float *cost, uint32_t *labels, uint32_t n, const uint32_t *region,
                         const uint32_t *cadj_ptr, const uint32_t *cadj_idx, const float *cwgt, const uint64_t *cptr,
                         const uint16_t *cview, const float *ccost, uint32_t *clabels, const uint32_t *params,
                         uint32_t *level_out, uint32_t *parent_out, uint32_t *swept, uint32_t *projected,
                         uint32_t *rejected, unsigned long long *slow_trees)
{
    const uint32_t root_div = params[0], seed = params[1], iter = params[2], group = params[3];
    if (!n || !F || n > F || iter == 0 || iter + 2 > MRF_SLOTS) return -2;
    const uint64_t nnz = ptr[F], cnnz = cptr[n];
    const uint32_t A = cadj_ptr[n];
    // the fine run's scratch (sized by F and nnz, as alloc_mrf makes it), with the 64 bytes of slack DevBuf::alloc gives
    std::vector<float> cost_al(nnz + 16), ccost_al(nnz + 16), wgt_al(A + 16), H(nnz + 16), hminp1(F), M(3 * (nnz + 16));
    std::vector<uint16_t> view_al(nnz + 32), cview_al(nnz + 32), olev(F), J(3 * (nnz + 16));
    std::copy(cost, cost + nnz, cost_al.begin());
    std::copy(view, view + nnz, view_al.begin());
    std::copy(ccost, ccost + cnnz, ccost_al.begin());
    std::copy(cview, cview + cnnz, cview_al.begin());
    std::copy(cwgt, cwgt + A, wgt_al.begin());
    std::vector<uint32_t> amin(F), level(F), lidx(F), clidx(n), order(F), pos(F, 0xFFFFFFFFu), queue(3 * (size_t)F + 1, 0u),
        ctl(CTL_WORDS, 0u), state(ST_WORDS, 0u), par(F), snap(2 * (size_t)F);
    std::vector<uint2> tjoin(F);
    std::vector<uint4> ttab(F), adj4(F), cadj4(n), rec(3 * (size_t)F);
    std::vector<unsigned long long> efix(MRF_SLOTS, 0ull);
    for (uint32_t v = 0; v < F; ++v) lidx[v] = label_pos(ptr, view, v, labels[v]);
    for (uint32_t r = 0; r < n; ++r) clidx[r] = label_pos(cptr, cview, r, clabels[r]);   // k_ml_lidx
    const uint32_t words = (K + 1 + 31) / 32;
    const uint32_t mask_words = (K == 0 || words > (uint32_t)MAX_MASK_WORDS) ? 0 : words;
    uint32_t maxn = 0;
    for (uint32_t v = 0; v < F; ++v) maxn = std::max<uint32_t>(maxn, (uint32_t)(ptr[v + 1] - ptr[v]));
    uint32_t tree_cap = std::min(1024u, std::max(16u, (maxn + 15u) & ~15u));
    if (params[4] >= 16) tree_cap = std::min(1024u, params[4] & ~15u);
    const uint32_t tree_smem = (uint32_t)TREE_WARPS * (32u / group) * tree_group_bytes(tree_cap, mask_words);
    if (tree_smem > sizeof(tree_dyn)) return -2;
    Mrf m;   // make_mrf
    m.F = F; m.nb = 0; m.ne = F;
    m.adj_ptr = adj_ptr; m.adj_idx = adj_idx; m.adj4 = adj4.data(); m.wgt = nullptr;
    m.ptr = ptr; m.view = view_al.data(); m.cost = cost_al.data();
    m.H = H.data(); m.hminp1 = hminp1.data(); m.amin = amin.data(); m.level = level.data();
    m.labels = labels; m.lidx = lidx.data();
    m.order = order.data(); m.olev = olev.data(); m.pos = pos.data();
    m.tjoin = tjoin.data(); m.ttab = ttab.data();
    m.ctl = ctl.data(); m.state = state.data();
    m.queue = queue.data(); m.qstamp = queue.data() + 2 * (size_t)F;
    m.efix = efix.data(); m.dbg = nullptr;
    m.K = K; m.mask_words = mask_words;
    m.part_size = F;
    m.rounds = 16;   // not read by the spanning kernels
    m.seed = seed; m.iter = iter;
    m.rdiv = 0;
    m.tree_smem = tree_smem;
    m.rec = reinterpret_cast<NodeRec *>(rec.data()); m.M = M.data(); m.J = J.data(); m.mstride = nnz + 16; m.tree_cap = tree_cap;
    m.par = par.data(); m.snap = snap.data(); m.snap_lidx = snap.data() + F;
    Mrf cm = m;   // make_coarse_mrf
    cm.F = n; cm.nb = 0; cm.ne = n;
    cm.adj_ptr = cadj_ptr; cm.adj_idx = cadj_idx; cm.adj4 = cadj4.data(); cm.wgt = wgt_al.data();
    cm.ptr = cptr; cm.view = cview_al.data(); cm.cost = ccost_al.data();
    cm.labels = clabels; cm.lidx = clidx.data();
    cm.part_size = n;
    if (root_div == 0) cm.rdiv = 0;
    else { uint32_t cap = n / 8u; if (cap < 1u) cap = 1u; cm.rdiv = root_div < cap ? root_div : cap; }
    emul::launch_serial((F + 255) / 256, 256, [&] { k_build_adj4(F, adj_ptr, adj_idx, adj4.data()); });
    emul::launch_serial((n + 255) / 256, 256, [&] { k_build_adj4(n, cadj_ptr, cadj_idx, cadj4.data()); });
    if (!emul::launch(2, 256, [&] { k_energy(m, m.efix + iter - 1); })) return -1;   // the energy before the step
    if (!emul::launch(1, FOREST_THREADS, [&] { k_forest<true>(cm, 1); })) return -1;
    emul::launch_serial((n + 255) / 256, 256, [&] { k_tree_prep<true>(cm); });
    bool ok;
    switch (group) {
        case 4: ok = emul::launch(1, TREE_THREADS, [&] { k_tree<4, 3, true, true>(cm); }); break;
        case 8: ok = emul::launch(1, TREE_THREADS, [&] { k_tree<8, 3, true, true>(cm); }); break;
        case 16: ok = emul::launch(1, TREE_THREADS, [&] { k_tree<16, 3, true, true>(cm); }); break;
        case 32: ok = emul::launch(1, TREE_THREADS, [&] { k_tree<32, 3, true, true>(cm); }); break;
        default: return -2;
    }
    if (!ok) return -1;
    std::copy(clabels, clabels + n, swept);
    std::copy(level.begin(), level.begin() + n, level_out);
    std::copy(par.begin(), par.begin() + n, parent_out);
    project(F, region, clabels, ptr, view, labels, lidx.data());
    std::copy(labels, labels + F, projected);
    if (!emul::launch(2, 256, [&] { k_energy(m, m.efix + iter); })) return -1;
    emul::launch_serial(1, 1, [&] { k_accept(m, iter); });
    emul::launch_serial(2, 256, [&] { k_restore(cm); });
    emul::launch_serial(1, 1, [&] { k_step_count(m); });
    if (!ctl[CTL_KEEP]) project(F, region, clabels, ptr, view, labels, lidx.data());
    *rejected = ctl[CTL_REJECT];
    if (state[ST_STEPS] != 1u || state[ST_STEP_REJ] != *rejected || state[ST_REJECTED] != *rejected) return -3;
    if (*rejected && efix[iter] != efix[iter - 1]) return -3;
    for (uint32_t r = 0; r < n; ++r)   // the coarse label positions went with the labels
        if (cptr[r + 1] > cptr[r] && (uint32_t)cview[cptr[r] + clidx[r]] + 1u != clabels[r]) return -3;
    if (slow_trees) *slow_trees = state[ST_SLOW];
    return 0;
}

}  // extern "C"
