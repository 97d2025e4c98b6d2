// tests/cpp/emul_mrf_spanning.cpp -- fiber emulation (cuda_fiber.h) of one spanning-tree iteration of csrc/mrf.cu, as
// enqueue_spanning_iteration drives it: k_build_adj4, k_forest<true>, k_tree_prep<true>, k_tree<G, 3, false, true> (fast
// path and the global-memory recursion), k_energy, k_accept and k_restore.  mrf_kernels.inc is the same cut of mrf.cu that
// tests/test_cuda_emulation.py makes.
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

extern "C" {

// params: [root_div, seed, iteration (>= 1), group (4 / 8 / 16 / 32), longest list the k_tree scratch holds (< 16: the
// longest list of the input)].  labels: in = current labels (0 = unseen face), out = after the iteration.  level, parent:
// [F] out.  swept: [F] out, the labels of the DP before acceptance.  rejected: out, k_accept's decision.
// Returns 0, -1 when a launch hung, -2 on bad parameters, -3 / -4 when the decision, the energy or the label positions
// after k_restore are inconsistent.
int emul_spanning_iteration(uint32_t n, uint32_t K, const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint64_t *ptr,
                            const uint16_t *view, const float *cost, const uint32_t *params, uint32_t *labels,
                            uint32_t *level_out, uint32_t *parent_out, uint32_t *swept, uint32_t *rejected,
                            unsigned long long *slow_trees)
{
    const uint32_t root_div = params[0], seed = params[1], iter = params[2], group = params[3];
    if (!n || iter == 0 || iter + 2 > MRF_SLOTS) return -2;
    const uint64_t nnz = ptr[n];
    // the 64 bytes of slack DevBuf::alloc gives every device array
    std::vector<float> cost_al(nnz + 16), H(nnz + 16), hminp1(n), M(3 * (nnz + 16));
    std::vector<uint16_t> view_al(nnz + 32), olev(n), J(3 * (nnz + 16));
    std::copy(cost, cost + nnz, cost_al.begin());
    std::copy(view, view + nnz, view_al.begin());
    std::vector<uint32_t> amin(n), level(n), lidx(n), order(n), pos(n, 0xFFFFFFFFu), queue(3 * (size_t)n + 1, 0u),
        ctl(CTL_WORDS, 0u), state(ST_WORDS, 0u), par(n), snap(2 * (size_t)n);
    std::vector<uint2> tjoin(n);
    std::vector<uint4> ttab(n), adj4(n), rec(3 * (size_t)n);
    std::vector<unsigned long long> efix(MRF_SLOTS, 0ull);
    for (uint32_t v = 0; v < n; ++v) {   // position of the current label
        uint32_t k = 0;
        while (ptr[v] + k < ptr[v + 1] && (uint32_t)view[ptr[v] + k] + 1u != labels[v]) ++k;
        lidx[v] = ptr[v + 1] > ptr[v] ? k : 0u;
    }
    const uint32_t words = (K + 1 + 31) / 32;
    const uint32_t mask_words = (K == 0 || words > (uint32_t)MAX_MASK_WORDS) ? 0 : words;
    uint32_t maxn = 0;
    for (uint32_t v = 0; v < n; ++v) maxn = std::max<uint32_t>(maxn, (uint32_t)(ptr[v + 1] - ptr[v]));
    uint32_t tree_cap = std::min(1024u, std::max(16u, (maxn + 15u) & ~15u));
    if (params[4] >= 16) tree_cap = std::min(1024u, params[4] & ~15u);
    const uint32_t tree_smem = (uint32_t)TREE_WARPS * (32u / group) * tree_group_bytes(tree_cap, mask_words);
    if (tree_smem > sizeof(tree_dyn)) return -2;
    Mrf m;
    m.F = n; m.nb = 0; m.ne = n;
    m.adj_ptr = adj_ptr; m.adj_idx = adj_idx; m.adj4 = adj4.data(); m.wgt = nullptr;
    m.ptr = ptr; m.view = view_al.data(); m.cost = cost_al.data();
    m.H = H.data(); m.hminp1 = hminp1.data(); m.amin = amin.data(); m.level = level.data();
    m.labels = labels; m.lidx = lidx.data();
    m.order = order.data(); m.olev = olev.data(); m.pos = pos.data();
    m.tjoin = tjoin.data(); m.ttab = ttab.data();
    m.ctl = ctl.data(); m.state = state.data();
    m.queue = queue.data(); m.qstamp = queue.data() + 2 * (size_t)n;
    m.efix = efix.data(); m.dbg = nullptr;
    m.K = K; m.mask_words = mask_words;
    m.part_size = n;
    m.rounds = 16;   // not read by the spanning kernels
    if (root_div == 0) m.rdiv = 0;
    else { uint32_t cap = n / 8u; if (cap < 1u) cap = 1u; m.rdiv = root_div < cap ? root_div : cap; }
    m.seed = seed; m.iter = iter;
    m.tree_smem = tree_smem;
    m.rec = reinterpret_cast<NodeRec *>(rec.data()); m.M = M.data(); m.J = J.data(); m.mstride = nnz + 16; m.tree_cap = tree_cap;
    m.par = par.data(); m.snap = snap.data(); m.snap_lidx = snap.data() + n;
    emul::launch_serial((n + 255) / 256, 256, [&] { k_build_adj4(n, adj_ptr, adj_idx, adj4.data()); });
    if (!emul::launch(2, 256, [&] { k_energy(m, m.efix + iter - 1); })) return -1;   // the energy before the iteration
    if (!emul::launch(1, FOREST_THREADS, [&] { k_forest<true>(m, 1); })) return -1;
    emul::launch_serial((n + 255) / 256, 256, [&] { k_tree_prep<true>(m); });
    bool ok;
    switch (group) {
        case 4: ok = emul::launch(1, TREE_THREADS, [&] { k_tree<4, 3, false, true>(m); }); break;
        case 8: ok = emul::launch(1, TREE_THREADS, [&] { k_tree<8, 3, false, true>(m); }); break;
        case 16: ok = emul::launch(1, TREE_THREADS, [&] { k_tree<16, 3, false, true>(m); }); break;
        case 32: ok = emul::launch(1, TREE_THREADS, [&] { k_tree<32, 3, false, true>(m); }); break;
        default: return -2;
    }
    if (!ok) return -1;
    std::copy(labels, labels + n, swept);
    if (!emul::launch(2, 256, [&] { k_energy(m, m.efix + iter); })) return -1;
    emul::launch_serial(1, 1, [&] { k_accept(m, iter); });
    emul::launch_serial(2, 256, [&] { k_restore(m); });
    std::copy(level.begin(), level.end(), level_out);
    std::copy(par.begin(), par.end(), parent_out);
    *rejected = ctl[CTL_REJECT];
    if (state[ST_REJECTED] != *rejected || (*rejected && efix[iter] != efix[iter - 1])) return -3;
    for (uint32_t v = 0; v < n; ++v)   // the label positions went with the labels
        if (ptr[v + 1] > ptr[v] && (uint32_t)view[ptr[v] + lidx[v]] + 1u != labels[v]) return -4;
    if (slow_trees) *slow_trees = state[ST_SLOW];
    return 0;
}

}  // extern "C"
