// mrf.cu -- K5-K7: pairwise-Potts MRF view selection on the device.
//
// Replaces tex::view_selection's call into mapMAP (libs/tex/view_selection.cpp:84-118); the model
// (label sets, unaries, Potts edges between seen faces) follows view_selection.cpp:26-82.
// Solver = block coordinate descent over induced forests with exact min-sum DP, the algorithm
// defined in oracle/mrf.c; this file reproduces it bit for bit:
//   * forest sampling is order independent (hash priorities, level-synchronous rounds)
//   * messages are summed in adjacency order in fp32 (no FMA: additions and minima only)
//   * the energy used for termination is 32.32 fixed point, summed with integer atomics.
//
// Execution (one iteration = 5 launches, NO host round trip: the stop rule is evaluated on the device
// and the host only polls a pinned flag a few iterations behind the launches it has queued):
//   k_forest   persistent cooperative kernel: root selection, `rounds` growth rounds on a frontier,
//              separated by grid.sync().  Every node that joins records (tree, slot) -- the tree of its
//              parent and its arrival number in that tree -- and adds its label count to the tree's
//              totals, so that the kernel can lay the forest out TREE BY TREE (levels ascending inside
//              a tree) without any sort: one block-aggregated allocation pass + one scatter pass.
//   k_tree_prep + k_tree<G>  the trees of an induced forest do not touch each other (every edge that leaves a tree
//              ends at a node whose label is fixed in this iteration), so the whole min-sum DP of a tree -- bottom-up
//              messages AND top-down assignment -- runs inside ONE warp, streamed through L2 without staging and
//              without block- or grid-wide barriers (see the comment above k_tree_prep).
//   k_energy   fixed-point energy -> efix[t] on the device
//   k_stop     StopWhenReturnsDiminish (view_selection.cpp:84) on the device; once it fires, the
//              launches the host has already queued return immediately
// use_multilevel (oracle/mrf_multilevel.c): after the stop rule fires, mrf_multilevel.cu contracts every same-label region
// into one node and the same launches run on the contracted MRF with weighted Potts terms (k_tree<G, MINB, true>), each
// iteration projected back onto the faces before k_energy (run_multilevel).
// use_spanning_tree (oracle/mrf_spanning.c): a spanning phase before the first acyclic one.  k_forest<true> grows a BFS
// spanning forest from the same roots and records every node's parent in `par`; k_tree_prep<true> classifies neighbours by
// `par` (every non-tree neighbour is fixed at its label from the start of the iteration), and k_accept / k_restore undo an
// iteration that raised the energy.
// spanning_tree_multilevel_after_n_iterations = n (oracle/mrf_mapmap.c, texrecon's mapMAP control): inside the spanning
// phase, after every n spanning iterations, one multilevel step -- the contraction, ONE spanning iteration on the contracted
// MRF (k_forest<true>, k_tree_prep<true>, k_tree<G, MINB, true, true>), the projection, and k_accept on the fine energy
// (enqueue_multilevel_step).  The acyclic phase follows and stays the last one.
#include <cooperative_groups.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <memory>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace b2 {

namespace {

constexpr uint32_t LVL_NONE = 0xFFFFFFFFu;
constexpr uint32_t LVL_DEAD = 0xFFFFFFFEu;
constexpr uint32_t NO_NODE = 0xFFFFFFFFu;
constexpr int MAX_LEVELS = 1024;    // rounds + 1 must fit
constexpr int MAX_MASK_WORDS = 64;  // label bitmasks up to K = 2047 views, else binary search

__host__ __device__ __forceinline__ uint32_t mix32(uint32_t x)
{
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}
__host__ __device__ __forceinline__ uint32_t iter_seed(uint32_t seed, uint32_t t)
{
    return mix32(seed + 0x9E3779B9u * (t + 1u));
}
__device__ __forceinline__ uint32_t prio(uint32_t v, uint32_t seed_t) { return mix32(v ^ seed_t); }
__device__ __forceinline__ bool root_cand(uint32_t v, uint32_t seed_t, uint32_t rdiv)
{
    return mix32(prio(v, seed_t) ^ 0x68E31DA4u) % rdiv == 0;
}

struct NodeRec;
struct Mrf {
    uint32_t F, nb, ne;          // nodes, owned node range
    const uint32_t *adj_ptr, *adj_idx;
    const uint4 *adj4;           // compact adjacency: x,y,z = neighbours, w = degree (CSR if > 3)
    const uint64_t *ptr;
    const uint16_t *view;
    const float *cost;
    float *H, *hminp1;           // global-memory DP scratch (oversize / high-degree trees only)
    uint32_t *amin;
    uint32_t *level, *labels, *lidx;   // lidx = position of the current label in the node's list
    uint32_t *order;             // forest nodes, tree by tree, levels ascending inside a tree
    uint16_t *olev;              // level of order[i]
    uint32_t *pos;               // index of a node in order, NO_NODE outside the forest
    uint2 *tjoin;                // per node: (tree, arrival number in the tree)
    uint4 *ttab;                 // per tree: (nodes | has a node of degree > 3 << 31, labels, first order index, message-row entries)
    uint32_t *ctl;               // per-iteration control block (zeroed before k_forest), see CTL_*
    uint32_t *state;             // per-run state, see ST_*
    uint32_t *queue, *qstamp;    // frontier lists [2][F] and push de-duplication stamps [F]
    unsigned long long *efix;    // [max_iterations + 1] fixed-point energies
    unsigned long long *dbg;     // optional phase timers of k_forest (B2TEX_FOREST_TIMING), else null
    uint32_t K, mask_words;
    uint32_t part_size, rounds, rdiv, seed, iter;
    uint32_t tree_smem;          // dynamic shared memory of k_tree (bytes)
    NodeRec *rec;                // per forest node, in `order` layout (k_tree_prep)
    float *M;                    // [3][mstride] messages child -> parent, per adjacency slot, at the parent's row positions
    uint16_t *J;                 // [3][mstride] position of that label in the child's list if the child should copy it, else 0xFFFF
    size_t mstride;
    uint32_t tree_cap;           // longest label list the shared-memory scratch of k_tree holds
    const float *wgt;            // Potts weight per adjacency slot (the contracted MRF of mrf_multilevel.cu), read by k_tree<.., true>
    uint32_t *par;               // spanning forests: parent of every node, NO_NODE for roots and nodes outside the forest
    uint32_t *snap, *snap_lidx;  // spanning forests: labels and label positions at the start of the iteration
};
// control block layout (uint32 words)
constexpr int CTL_QN = 0;                        // [MAX_LEVELS+1] frontier sizes per round
constexpr int CTL_NROOTS = MAX_LEVELS + 8;       // trees of this iteration
constexpr int CTL_CURSOR = MAX_LEVELS + 9;       // forest nodes laid out so far
constexpr int CTL_CLAIM = MAX_LEVELS + 10;       // k_tree: next unclaimed tree
constexpr int CTL_REJECT = MAX_LEVELS + 11;      // spanning iteration: k_accept rejected it, k_restore brings the labels back
constexpr int CTL_MAXPRIO = MAX_LEVELS + 12;     // 64-bit, 8-byte aligned
constexpr int CTL_KEEP = MAX_LEVELS + 14;        // multilevel step: nonzero unless it was rejected (skips the re-projection)
constexpr int CTL_WORDS = MAX_LEVELS + 32;
// run state (uint32 words)
constexpr int ST_STOP = 0;      // 0 while running, else the iteration the stop rule fired in
constexpr int ST_DONE = 1;      // last iteration whose energy is final
constexpr int ST_BAD = 2;       // labels > K found by k_label_check
constexpr int ST_UNSEEN = 3;    // faces with label 0
constexpr int ST_FNODES = 4;    // 64-bit: forest nodes summed over the iterations (roofline accounting)
constexpr int ST_FNNZ = 6;      // 64-bit: labels of forest nodes summed over the iterations
constexpr int ST_SLOW = 8;      // trees that went through global memory
constexpr int ST_ERR = 9;       // cross-GPU barrier timeouts (a peer did not arrive)
constexpr int ST_REJECTED = 10; // spanning iterations and multilevel steps that raised the energy and were undone
constexpr int ST_STEPS = 11;    // multilevel steps of the spanning phase
constexpr int ST_STEP_REJ = 12; // of those, the ones that were undone
constexpr int ST_WORDS = 16;

__device__ __forceinline__ bool same_part(const Mrf &m, uint32_t a, uint32_t b)
{
    if (m.part_size >= m.F) return true;  // single partition: no integer divisions on the hot path
    return a / m.part_size == b / m.part_size;
}
__device__ __forceinline__ bool owned(const Mrf &m, uint32_t v) { return v >= m.nb && v < m.ne; }
__device__ __forceinline__ bool local_pair(const Mrf &m, uint32_t v, uint32_t w)
{
    return owned(m, w) && same_part(m, v, w);
}

// Neighbour list of one node.  Face graphs of manifold meshes have degree <= 3: one 16-byte load
// replaces the adj_ptr -> adj_idx dependent chain; larger degrees fall back to the CSR arrays.
struct Nb { uint32_t deg, x, y, z, base; };
__device__ __forceinline__ Nb load_nb(const Mrf &m, uint32_t v)
{
    const uint4 a = __ldg(m.adj4 + v);
    Nb n; n.deg = a.w; n.x = a.x; n.y = a.y; n.z = a.z;
    n.base = a.w > 3 ? m.adj_ptr[v] : 0;
    return n;
}
__device__ __forceinline__ uint32_t nb_at(const Mrf &m, const Nb &n, uint32_t i)
{
    if (n.deg <= 3) return i == 0 ? n.x : (i == 1 ? n.y : n.z);
    return m.adj_idx[n.base + i];
}

// longest label list of the owned faces
__global__ void __launch_bounds__(256) k_max_labels(const uint64_t *__restrict__ ptr, uint32_t nb, uint32_t ne, uint32_t *out)
{
    uint32_t mx = 0;
    for (uint32_t v = nb + blockIdx.x * blockDim.x + threadIdx.x; v < ne; v += gridDim.x * blockDim.x)
        mx = max(mx, (uint32_t)(ptr[v + 1] - ptr[v]));
    mx = __reduce_max_sync(0xffffffffu, mx);
    if ((threadIdx.x & 31) == 0 && mx) atomicMax(out, mx);
}

__global__ void __launch_bounds__(256) k_build_adj4(uint32_t F, const uint32_t *__restrict__ adj_ptr,
                                                    const uint32_t *__restrict__ adj_idx, uint4 *adj4)
{
    uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= F) return;
    uint32_t a0 = adj_ptr[v], d = adj_ptr[v + 1] - a0;
    uint4 r = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, d);
    if (d <= 3) {
        if (d > 0) r.x = adj_idx[a0];
        if (d > 1) r.y = adj_idx[a0 + 1];
        if (d > 2) r.z = adj_idx[a0 + 2];
    }
    adj4[v] = r;
}

// ---- shared-memory / async-copy primitives (the host emulation replaces this block) ----
__device__ __forceinline__ unsigned long long global_timer_ns()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// ---- end of primitives ----

template <int G>
__global__ void __launch_bounds__(256) k_init_labels(Mrf m)
{
    const uint32_t lane = threadIdx.x & (G - 1);
    const uint32_t gpw = blockDim.x / G;
    for (uint32_t base = m.nb + blockIdx.x * gpw; base < m.ne; base += gridDim.x * gpw) {
        uint32_t v = base + threadIdx.x / G;
        bool act = v < m.ne;
        uint64_t p0 = act ? m.ptr[v] : 0, p1 = act ? m.ptr[v + 1] : 0;
        float bh = INFINITY;
        uint32_t bk = 0xFFFFFFFFu;
        for (uint64_t k = p0 + lane; k < p1; k += G) {
            float c = m.cost[k];
            if (c < bh) { bh = c; bk = (uint32_t)(k - p0); }
        }
        __syncwarp();
        for (int s = G / 2; s; s >>= 1) {
            float oh = __shfl_xor_sync(0xffffffffu, bh, s);
            uint32_t ok = __shfl_xor_sync(0xffffffffu, bk, s);
            if (oh < bh || (oh == bh && ok < bk)) { bh = oh; bk = ok; }
        }
        if (act && lane == 0) {
            m.labels[v] = (p1 > p0) ? (uint32_t)m.view[p0 + bk] + 1u : 0u;
            m.lidx[v] = (p1 > p0) ? bk : 0u;
        }
    }
}

// position of label `lab` (= view+1) in node w's sorted list, or -1
__device__ __forceinline__ long long find_label(const Mrf &m, uint32_t w, uint32_t lab)
{
    uint64_t lo = m.ptr[w], end = m.ptr[w + 1], hi = end;
    while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        uint32_t l = (uint32_t)m.view[mid] + 1u;
        if (l < lab) lo = mid + 1; else hi = mid;
    }
    if (lo < end && (uint32_t)m.view[lo] + 1u == lab) return (long long)lo;
    return -1;
}

// ---- forest sampling + tree layout, one persistent cooperative launch -----------------------------
__device__ __forceinline__ uint32_t count_in_forest(const Mrf &m, uint32_t v, uint32_t r)
{
    uint32_t c = 0;
    const Nb nb = load_nb(m, v);
    for (uint32_t i = 0; i < nb.deg; ++i) {
        uint32_t w = nb_at(m, nb, i);
        if (local_pair(m, v, w) && __ldcg(m.level + w) < r) ++c;
    }
    return c;
}

constexpr int FOREST_THREADS = 1024;
// growth rounds at most: `rounds` for induced forests, the bound alloc_mrf puts on `rounds` for spanning forests
template <bool S>
__device__ __forceinline__ uint32_t growth_rounds(const Mrf &m) { return S ? (uint32_t)(MAX_LEVELS - 2) : m.rounds; }
// S: spanning forest (oracle/mrf_spanning.c) -- every queued undecided node joins, under its strongest neighbour of the
// previous level (recorded in m.par), until a round adds nobody or after MAX_LEVELS - 2 rounds; round 0 also snapshots the
// labels for k_restore
template <bool S = false>
__global__ void __launch_bounds__(FOREST_THREADS, 1) k_forest(Mrf m, int build_trees)
{
    cg::grid_group grid = cg::this_grid();
    if (__ldcg(m.state + ST_STOP)) return;  // the stop rule fired in an earlier iteration (grid-uniform)
    __shared__ uint32_t s_cnt, s_base, s_warp[FOREST_THREADS / 32];
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
    unsigned long long t_prev = 0;
    auto stamp = [&](int slot) {   // diagnostic: nanoseconds per phase, accumulated over the iterations
        if (m.dbg && tid == 0) {
            const unsigned long long t = global_timer_ns();
            if (t_prev) m.dbg[slot] += t - t_prev;
            t_prev = t;
        }
    };
    stamp(0);
    const uint32_t seed_t = iter_seed(m.seed, m.iter);
    const uint32_t n_own = m.ne - m.nb;
    unsigned long long *maxprio = reinterpret_cast<unsigned long long *>(m.ctl + CTL_MAXPRIO);

    if (m.rdiv == 0) {  // single-root mode: the seen node with the largest priority
        unsigned long long key = 0;
        for (uint32_t v = m.nb + tid; v < m.ne; v += nth)
            if (m.labels[v] != 0) {
                unsigned long long k = (((unsigned long long)prio(v, seed_t)) << 1) | 1ull;
                key = k > key ? k : key;
            }
        for (int s = 16; s; s >>= 1) {
            unsigned long long o = __shfl_xor_sync(0xffffffffu, key, s);
            key = o > key ? o : key;
        }
        if ((threadIdx.x & 31) == 0 && key) atomicMax(maxprio, key);
        grid.sync();
    }
    // round 0: eligibility and roots (full scan, once).  Roots open a tree: compact tree numbers come from one
    // global atomic per block and pass (block-aggregated), not one per root.
    for (uint32_t base = blockIdx.x * blockDim.x; base < n_own; base += nth) {  // block-uniform trip count
        const uint32_t v = m.nb + base + threadIdx.x;
        const bool valid = v < m.ne;
        uint32_t lvl = LVL_DEAD;
        if (valid && m.labels[v] != 0) {
            const uint32_t pv = prio(v, seed_t);
            bool eligible = true, is_root;
            if (m.rdiv) is_root = root_cand(v, seed_t, m.rdiv);
            else is_root = __ldcg(maxprio) == ((((unsigned long long)pv) << 1) | 1ull);
            const Nb nb = load_nb(m, v);
            for (uint32_t i = 0; i < nb.deg; ++i) {
                uint32_t w = nb_at(m, nb, i);
                if (m.labels[w] == 0) continue;
                if (!local_pair(m, v, w)) { if (prio(w, seed_t) > pv) eligible = false; continue; }
                if (m.rdiv && is_root && root_cand(w, seed_t, m.rdiv) && prio(w, seed_t) > pv) is_root = false;
            }
            lvl = !eligible ? LVL_DEAD : (is_root ? 0u : LVL_NONE);
        }
        if (valid) { m.level[v] = lvl; if (build_trees) m.pos[v] = NO_NODE; }
        if constexpr (S) {
            if (valid) { m.par[v] = NO_NODE; m.snap[v] = m.labels[v]; m.snap_lidx[v] = m.lidx[v]; }
        }
        if (build_trees) {
            const bool is_root = valid && lvl == 0u;
            if (threadIdx.x == 0) s_cnt = 0;
            __syncthreads();
            uint32_t my = 0;
            if (is_root) my = atomicAdd(&s_cnt, 1u);
            __syncthreads();
            if (threadIdx.x == 0 && s_cnt) s_base = atomicAdd(&m.ctl[CTL_NROOTS], s_cnt);
            __syncthreads();
            if (is_root) {
                const uint32_t j = s_base + my;
                const uint32_t nl = (uint32_t)(m.ptr[v + 1] - m.ptr[v]);
                m.ttab[j] = make_uint4(1u | (__ldg(&m.adj4[v].w) > 3u ? 0x80000000u : 0u), nl, 0u, 0u);
                m.tjoin[v] = make_uint2(j, 0u);
            }
        }
    }
    grid.sync();
    stamp(1);   // round 0
    // Growth rounds on a FRONTIER instead of full scans.  Only an undecided node with >= 1 forest
    // neighbour can change state in a round, and such a node is either newly adjacent to a node that
    // joined in the previous round (pushed by that node) or a candidate that lost and re-queues
    // itself.  The evaluated set equals the set a full scan would act on, so levels are identical to
    // oracle/mrf.c; list order is irrelevant.  qstamp de-duplicates pushes (unique per iteration+round).
    const uint32_t stamp_base = m.iter * 2048u;
    // Appending to the next frontier: one global atomic per BLOCK and pass (all pushes of a round go to the same
    // counter, so one atomic per push serialises a round on that counter).  A thread collects its pushes first.
    constexpr int PEND = 4;
    uint32_t pend[PEND], np = 0;
    auto push_direct = [&](uint32_t w, uint32_t round) {
        const uint32_t at = atomicAdd(&m.ctl[CTL_QN + round], 1u);
        m.queue[(size_t)(round & 1u) * m.F + at] = w;
    };
    auto push = [&](uint32_t w, uint32_t round) {
        if (atomicExch(m.qstamp + w, stamp_base + round) == stamp_base + round) return;   // already queued
        if (np < (uint32_t)PEND) pend[np++] = w; else push_direct(w, round);
    };
    auto flush = [&](uint32_t round) {   // block-wide: every thread of the block calls it the same number of times
        if (threadIdx.x == 0) s_cnt = 0;
        __syncthreads();
        const uint32_t off = np ? atomicAdd(&s_cnt, np) : 0u;
        __syncthreads();
        if (threadIdx.x == 0 && s_cnt) s_base = atomicAdd(&m.ctl[CTL_QN + round], s_cnt);
        __syncthreads();
        for (uint32_t i = 0; i < np; ++i) m.queue[(size_t)(round & 1u) * m.F + s_base + off + i] = pend[i];
        np = 0;
    };
    for (uint32_t base = blockIdx.x * blockDim.x; base < n_own; base += nth) {  // seed: undecided neighbours of the roots
        const uint32_t v = m.nb + base + threadIdx.x;
        if (v < m.ne && __ldcg(m.level + v) == 0u) {
            const Nb nb = load_nb(m, v);
            for (uint32_t i = 0; i < nb.deg; ++i) {
                uint32_t w = nb_at(m, nb, i);
                if (local_pair(m, v, w) && __ldcg(m.level + w) == LVL_NONE) push(w, 1u);
            }
        }
        flush(1u);
    }
    grid.sync();
    stamp(2);   // frontier seeding
    for (uint32_t r = 1; r <= growth_rounds<S>(m); ++r) {
        const uint32_t n = __ldcg(m.ctl + CTL_QN + r);
        if constexpr (S) {
            if (n == 0) break;   // final since the last grid.sync(): grid-uniform
        }
        const uint32_t *q = m.queue + (size_t)(r & 1u) * m.F;
        for (uint32_t base = blockIdx.x * blockDim.x; base < n; base += nth) {   // block-uniform trip count
            const uint32_t qi = base + threadIdx.x;
            const uint32_t v = qi < n ? __ldcg(q + qi) : NO_NODE;
            if (v != NO_NODE && __ldcg(m.level + v) == LVL_NONE) {
                const Nb nb = load_nb(m, v);
                uint32_t c = 0, parent = NO_NODE;
                bool win = true;
                if constexpr (S) {   // a queued node has a neighbour of level r - 1 (and none lower): it joins
                    uint32_t pp = 0;
                    for (uint32_t i = 0; i < nb.deg; ++i) {
                        const uint32_t w = nb_at(m, nb, i);
                        if (!local_pair(m, v, w) || __ldcg(m.level + w) >= r) continue;
                        const uint32_t pw = prio(w, seed_t);
                        if (parent == NO_NODE || pw > pp) { parent = w; pp = pw; }
                    }
                    c = parent != NO_NODE ? 1u : 0u;
                } else if (nb.deg <= 3) {
                    // manifold degree: every load of a hop is issued before the first one is used (the round is a chain of
                    // dependent loads; two hops instead of up to eight round trips)
                    const uint32_t wn[3] = {nb.x, nb.y, nb.z};
                    uint32_t lw[3];
                    bool loc[3];
#pragma unroll
                    for (int i = 0; i < 3; ++i) {
                        loc[i] = (uint32_t)i < nb.deg && local_pair(m, v, wn[i]);
                        lw[i] = loc[i] ? __ldcg(m.level + wn[i]) : LVL_DEAD;
                    }
#pragma unroll
                    for (int i = 0; i < 3; ++i)
                        if (loc[i] && lw[i] < r) { ++c; parent = wn[i]; }
                    if (c == 1) {
                        const uint32_t pv = prio(v, seed_t);
                        bool cont[3];
                        uint4 a4[3];
#pragma unroll
                        for (int i = 0; i < 3; ++i) {   // undecided (or just joined) local neighbours that are not weaker
                            cont[i] = loc[i] && (lw[i] == LVL_NONE || lw[i] == r) && !(prio(wn[i], seed_t) < pv);
                            a4[i] = cont[i] ? __ldg(m.adj4 + wn[i]) : make_uint4(NO_NODE, NO_NODE, NO_NODE, 0u);
                        }
#pragma unroll
                        for (int i = 0; i < 3; ++i) {
                            if (!cont[i]) continue;
                            uint32_t cw = 0;
                            if (a4[i].w <= 3) {
                                const uint32_t xn[3] = {a4[i].x, a4[i].y, a4[i].z};
                                uint32_t lx[3];
#pragma unroll
                                for (int j = 0; j < 3; ++j)
                                    lx[j] = ((uint32_t)j < a4[i].w && local_pair(m, wn[i], xn[j])) ? __ldcg(m.level + xn[j]) : LVL_DEAD;
#pragma unroll
                                for (int j = 0; j < 3; ++j) cw += lx[j] < r ? 1u : 0u;
                            } else cw = count_in_forest(m, wn[i], r);
                            if (cw == 1) win = false;  // a stronger adjacent candidate: wait
                        }
                    }
                } else {
                    for (uint32_t i = 0; i < nb.deg; ++i) {
                        uint32_t w = nb_at(m, nb, i);
                        if (local_pair(m, v, w) && __ldcg(m.level + w) < r) { ++c; parent = w; }
                    }
                    if (c == 1) {
                        const uint32_t pv = prio(v, seed_t);
                        for (uint32_t i = 0; i < nb.deg && win; ++i) {
                            uint32_t w = nb_at(m, nb, i);
                            if (!local_pair(m, v, w)) continue;
                            uint32_t lw = __ldcg(m.level + w);
                            if (!(lw == LVL_NONE || lw == r)) continue;
                            if (prio(w, seed_t) < pv) continue;
                            if (count_in_forest(m, w, r) == 1) win = false;  // a stronger adjacent candidate: wait
                        }
                    }
                }
                if (c >= 2) m.level[v] = LVL_DEAD;
                else if (c == 1) {
                    if (win) {
                        m.level[v] = r;
                        if constexpr (S) m.par[v] = parent;
                        if (build_trees) {   // the parent joined in an earlier round: its (tree, slot) is final
                            const uint2 pj = __ldcg(m.tjoin + parent);
                            uint4 *te = m.ttab + pj.x;
                            const uint32_t slot = atomicAdd(&te->x, 1u) & 0x7FFFFFFFu;
                            atomicAdd(&te->y, (uint32_t)(m.ptr[v + 1] - m.ptr[v]));
                            atomicAdd(&te->w, (uint32_t)(m.ptr[parent + 1] - m.ptr[parent]));   // its message row: one entry per label of the parent
                            if (nb.deg > 3) atomicOr(&te->x, 0x80000000u);
                            m.tjoin[v] = make_uint2(pj.x, slot);
                        }
                        if (r < growth_rounds<S>(m))
                            for (uint32_t i = 0; i < nb.deg; ++i) {
                                uint32_t w = nb_at(m, nb, i);
                                if (local_pair(m, v, w) && __ldcg(m.level + w) == LVL_NONE) push(w, r + 1u);
                            }
                    } else if (r < growth_rounds<S>(m)) {
                        push(v, r + 1u);
                    }
                }
            }
            if (r < growth_rounds<S>(m)) flush(r + 1u);
        }
        grid.sync();
    }
    stamp(3);   // growth rounds
    if (!build_trees) return;

    // ---- lay the forest out tree by tree: arrival numbers grow with the rounds, so the nodes of a tree are
    // ---- sorted by level; which tree comes first in memory is irrelevant (block-aggregated allocation)
    const uint32_t nroots = __ldcg(m.ctl + CTL_NROOTS);
    for (uint32_t base = blockIdx.x * blockDim.x; base < nroots; base += nth) {
        const uint32_t j = base + threadIdx.x;
        const uint32_t cnt = j < nroots ? (__ldcg(&m.ttab[j].x) & 0x7FFFFFFFu) : 0u;
        uint32_t incl = cnt;
        for (int s = 1; s < 32; s <<= 1) {
            uint32_t o = __shfl_up_sync(0xffffffffu, incl, s);
            if ((int)(threadIdx.x & 31) >= s) incl += o;
        }
        if ((threadIdx.x & 31) == 31) s_warp[threadIdx.x >> 5] = incl;
        __syncthreads();
        if (threadIdx.x < 32) {
            uint32_t w = threadIdx.x < (uint32_t)(FOREST_THREADS / 32) ? s_warp[threadIdx.x] : 0u, wi = w;
            for (int s = 1; s < 32; s <<= 1) {
                uint32_t o = __shfl_up_sync(0xffffffffu, wi, s);
                if ((int)threadIdx.x >= s) wi += o;
            }
            if (threadIdx.x < (uint32_t)(FOREST_THREADS / 32)) s_warp[threadIdx.x] = wi - w;  // exclusive warp offsets
            if (threadIdx.x == 31) s_base = wi ? atomicAdd(&m.ctl[CTL_CURSOR], wi) : 0u;
        }
        __syncthreads();
        if (j < nroots) m.ttab[j].z = s_base + s_warp[threadIdx.x >> 5] + incl - cnt;
        __syncthreads();
    }
    grid.sync();
    stamp(4);   // tree allocation
    unsigned long long fn = 0, fz = 0;
    for (uint32_t v = m.nb + tid; v < m.ne; v += nth) {
        const uint32_t l = __ldcg(m.level + v);
        if (l > growth_rounds<S>(m)) continue;
        const uint2 tj = __ldcg(m.tjoin + v);
        const uint32_t idx = __ldcg(&m.ttab[tj.x].z) + tj.y;
        m.order[idx] = v;
        m.olev[idx] = (uint16_t)l;
        m.pos[v] = idx;
        fn += 1ull;
        fz += m.ptr[v + 1] - m.ptr[v];
    }
    for (int s = 16; s; s >>= 1) { fn += __shfl_xor_sync(0xffffffffu, fn, s); fz += __shfl_xor_sync(0xffffffffu, fz, s); }
    if ((threadIdx.x & 31) == 0 && fn) {
        atomicAdd(reinterpret_cast<unsigned long long *>(m.state + ST_FNODES), fn);
        atomicAdd(reinterpret_cast<unsigned long long *>(m.state + ST_FNNZ), fz);
    }
    stamp(5);   // scatter (thread 0's share)
}

// ---- min-sum DP of whole trees: one warp per tree, streamed through L2 ------------------------------------------------
// The trees of an induced forest do not touch each other (every edge that leaves a tree ends at a node whose label is
// fixed in this iteration), so a tree is solved by ONE warp from its leaves to its root and back, without any block- or
// grid-wide barrier; 32 resident warps per SM hide the latency of each other's loads.  Nothing of a tree is staged:
//   k_tree_prep  one thread per forest node writes a 48-byte record in forest order: row extents, the role of each of the
//                three neighbours (child / parent / fixed label / none) and where the node's message to its parent goes.
//                This takes the three-deep chain of dependent loads (order -> adjacency -> labels / positions -> parent's
//                adjacency) out of the serial path of the DP.
//   k_tree<G>    bottom-up, level by level, G lanes per node (32 / G nodes of one level at a time): h(l) = cost(l) + the
//                terms of the neighbours in adjacency order -- a child contributes its Potts message
//                min(h_c(l), hmin_c + 1), which the CHILD wrote into the message row of that adjacency slot at the
//                parent's row position (M[slot][ptr[parent] + k], one float per label of the parent), so the parent reads
//                it with the same coalesced index as its own costs -- then min / arg-min by two warp reductions.  The
//                node's own h row lives in a small shared-memory scratch only until its message is formed (binary search
//                of every label of the parent in the node's sorted label list).  Next to every message entry the child
//                leaves the position of that label in its own list if choosing it is optimal given the parent
//                (J[slot][...], 0xFFFF = "take the arg-min"), so the top-down pass is one thread per node: two loads.
// DRAM traffic per forest node: 6 B per label (cost + view, read once) + 6 B per label of its parent written (message +
// position; the read-back hits L2) + ~100 B of record, against the 14 B per label of a sweep through global memory
// tables (SURVEY 8d).  Trees with a node of degree > 3 or a label list longer than the scratch take the same recursion
// through the global tables H / hminp1 / amin (tree_solve_global).
constexpr int TREE_THREADS = 512;
constexpr int TREE_WARPS = TREE_THREADS / 32;
constexpr uint32_t TREE_SMEM_MAX = 200u * 1024u;   // dynamic shared memory every k_tree instance opts in to (bytes)
constexpr uint32_t NBR_SKIP = 0u, NBR_CHILD = 1u << 30, NBR_FIXED = 2u << 30, NBR_PARENT = 3u << 30;
constexpr uint32_t NBR_KIND = 3u << 30, NBR_ARG = ~NBR_KIND;

struct __align__(16) NodeRec {
    uint32_t v;          // node
    uint32_t n_lev;      // label count | level << 16
    uint64_t p0;         // first entry of the node's cost / view rows
    uint32_t nbr[3];     // per adjacency slot: kind | argument (FIXED: the label, PARENT: the parent node)
    uint32_t pslot_pn;   // adjacency slot of this node at its parent | label count of the parent << 16
    uint64_t pp0;        // first entry of the parent's rows
    uint32_t amin;       // written bottom-up: position of the node's best label given its subtree
    uint32_t pad;
};
static_assert(sizeof(NodeRec) == 48, "NodeRec layout");

// S: spanning forest -- children are the neighbours w with par[w] == v, the parent is par[v], every other seen neighbour
// is fixed at the label it has now (before k_tree writes any)
template <bool S = false>
__global__ void __launch_bounds__(256) k_tree_prep(Mrf m)
{
    if (__ldcg(m.state + ST_STOP)) return;
    const uint32_t total = __ldcg(m.ctl + CTL_CURSOR);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const uint32_t v = m.order[i];
    const uint64_t p0 = m.ptr[v];
    const uint32_t n = (uint32_t)(m.ptr[v + 1] - p0);
    const uint4 a4 = __ldg(m.adj4 + v);
    NodeRec r;
    r.v = v; r.n_lev = n | ((uint32_t)m.olev[i] << 16); r.p0 = p0;
    r.nbr[0] = r.nbr[1] = r.nbr[2] = NBR_SKIP;
    r.pslot_pn = 0; r.pp0 = 0; r.amin = 0; r.pad = 0;
    if (n > m.tree_cap) atomicOr(&m.ttab[m.tjoin[v].x].x, 0x80000000u);   // longer than the scratch: through global memory
    if (a4.w <= 3) {
        // all six neighbour loads first (independent), classification afterwards
        uint32_t xl[3] = {0u, 0u, 0u}, pl[3] = {NO_NODE, NO_NODE, NO_NODE}, wn[3] = {a4.x, a4.y, a4.z};
#pragma unroll
        for (int a = 0; a < 3; ++a)
            if ((uint32_t)a < a4.w && wn[a] != NO_NODE) { xl[a] = m.labels[wn[a]]; pl[a] = S ? m.par[wn[a]] : m.pos[wn[a]]; }
        const uint32_t pv = S ? m.par[v] : NO_NODE;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            if (xl[a] == 0u) continue;   // unseen faces carry no edges (view_selection.cpp:30,35)
            if constexpr (S) {   // pl = the neighbour's parent
                if (pl[a] == v) { r.nbr[a] = NBR_CHILD; continue; }
                if (wn[a] != pv) { r.nbr[a] = NBR_FIXED | xl[a]; continue; }
            } else {
                if (pl[a] == NO_NODE) { r.nbr[a] = NBR_FIXED | xl[a]; continue; }
                if (pl[a] > i) { r.nbr[a] = NBR_CHILD; continue; }   // a forest neighbour is in the same tree: deeper = child
            }
            const uint32_t w = wn[a];
            const uint4 b4 = __ldg(m.adj4 + w);
            const uint64_t q0 = m.ptr[w];
            const uint32_t pn = (uint32_t)(m.ptr[w + 1] - q0);
            const uint32_t ps = b4.x == v ? 0u : (b4.y == v ? 1u : 2u);
            r.nbr[a] = NBR_PARENT | w;
            r.pslot_pn = ps | (pn << 16);
            r.pp0 = q0;
        }
    }
    uint4 *dst = reinterpret_cast<uint4 *>(m.rec + i);
    const uint4 *src = reinterpret_cast<const uint4 *>(&r);
    dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2];
}

// first index of the run of equal levels that ends at `end` (exclusive), searched inside [a, end)
template <typename LevPtr>
__device__ __forceinline__ uint32_t level_run_begin(LevPtr lev, uint32_t a, uint32_t end, uint32_t lane)
{
    const uint32_t L = lev[end - 1];
    uint32_t s = end;
    for (;;) {
        const bool p = s > a + lane && lev[s - 1 - lane] == L;
        const uint32_t b = __ballot_sync(0xffffffffu, p);
        const uint32_t run = b == 0xFFFFFFFFu ? 32u : (uint32_t)__ffs((int)~b) - 1u;
        s -= run;
        if (run < 32u) break;
    }
    return s;
}
// end (exclusive) of the run of equal levels that starts at `s`, searched inside [s, b)
template <typename LevPtr>
__device__ __forceinline__ uint32_t level_run_end(LevPtr lev, uint32_t s, uint32_t b, uint32_t lane)
{
    const uint32_t L = lev[s];
    uint32_t e = s;
    for (;;) {
        const bool p = e + lane < b && lev[e + lane] == L;
        const uint32_t bits = __ballot_sync(0xffffffffu, p);
        const uint32_t run = bits == 0xFFFFFFFFu ? 32u : (uint32_t)__ffs((int)~bits) - 1u;
        e += run;
        if (run < 32u) break;
    }
    return e;
}

// Potts weight of adjacency slot q of node v: 1 on the face graph, the number of fine edges on a contracted graph
template <bool W>
__device__ __forceinline__ float slot_weight(const Mrf &m, uint32_t v, uint32_t q)
{
    if constexpr (W) return m.wgt[m.adj_ptr[v] + q];
    else return 1.0f;
}

// the same recursion through global memory: any degree, any size (one node at a time, 32 lanes over its labels).
// S: a spanning forest, classified by m.par as k_tree_prep<true> does; fixed labels come from the snapshot, because the
// top-down passes of other warps write m.labels meanwhile and a spanning tree has edges to other trees.  W and S together:
// the spanning forest of a contracted MRF, the weight of the edge to the parent is that of the slot holding par[v].
template <bool W, bool S = false>
__device__ void tree_solve_global(const Mrf &m, uint32_t start, uint32_t cnt, uint32_t lane)
{
    const uint16_t *lev = m.olev + start;
    for (uint32_t end = cnt; end > 0;) {
        const uint32_t s = level_run_begin(lev, 0u, end, lane);
        for (uint32_t i = s; i < end; ++i) {
            const uint32_t v = m.order[start + i];
            const uint64_t p0 = m.ptr[v], p1 = m.ptr[v + 1];
            const Nb nb = load_nb(m, v);
            float wpar = 1.0f;   // weight of the edge to the parent
            if constexpr (W && S) {
                const uint32_t pv = m.par[v];
                for (uint32_t q = 0; q < nb.deg; ++q)
                    if (nb_at(m, nb, q) == pv) wpar = slot_weight<W>(m, v, q);
            } else if constexpr (W) {
                for (uint32_t q = 0; q < nb.deg; ++q) {
                    const uint32_t w = nb_at(m, nb, q);
                    const uint32_t pw = m.pos[w];
                    if (m.labels[w] != 0 && pw != NO_NODE && pw < start + i) wpar = slot_weight<W>(m, v, q);
                }
            }
            float bh = INFINITY;
            uint32_t bk = 0xFFFFFFFFu;
            const uint32_t par_v = S ? m.par[v] : NO_NODE;
            for (uint64_t k = p0 + lane; k < p1; k += 32) {
                const uint32_t lab = (uint32_t)m.view[k] + 1u;
                float h = m.cost[k];
                for (uint32_t q = 0; q < nb.deg; ++q) {
                    const uint32_t w = nb_at(m, nb, q);
                    if constexpr (S) {
                        const uint32_t x = m.snap[w];
                        if (x == 0) continue;
                        if (__ldcg(m.par + w) == v) {   // child
                            float msg = __ldcg(m.hminp1 + w);
                            const long long j = find_label(m, w, lab);
                            if (j >= 0) { const float hw = __ldcg(m.H + j); if (hw < msg) msg = hw; }
                            h = h + msg;
                        } else if (w != par_v) {
                            h = h + (lab != x ? slot_weight<W>(m, v, q) : 0.0f);
                        }
                        continue;
                    }
                    const uint32_t x = m.labels[w];
                    if (x == 0) continue;
                    const uint32_t pw = m.pos[w];
                    if (pw != NO_NODE) {
                        if (pw > start + i) {  // child
                            float msg = __ldcg(m.hminp1 + w);
                            const long long j = find_label(m, w, lab);
                            if (j >= 0) { const float hw = __ldcg(m.H + j); if (hw < msg) msg = hw; }
                            h = h + msg;
                        }
                    } else {
                        h = h + (lab != x ? slot_weight<W>(m, v, q) : 0.0f);
                    }
                }
                m.H[k] = h;
                if (h < bh) { bh = h; bk = (uint32_t)(k - p0); }
            }
            for (int sft = 16; sft; sft >>= 1) {
                const float oh = __shfl_xor_sync(0xffffffffu, bh, sft);
                const uint32_t ok = __shfl_xor_sync(0xffffffffu, bk, sft);
                if (oh < bh || (oh == bh && ok < bk)) { bh = oh; bk = ok; }
            }
            if (lane == 0) { m.hminp1[v] = bh + wpar; m.amin[v] = bk; }
        }
        __syncwarp();
        end = s;
    }
    for (uint32_t s = 0; s < cnt;) {
        const uint32_t e = level_run_end(lev, s, cnt, lane);
        for (uint32_t i = s + lane; i < e; i += 32) {
            const uint32_t v = m.order[start + i];
            uint32_t bk = __ldcg(m.amin + v);
            const Nb nb = load_nb(m, v);
            if constexpr (S) {
                const uint32_t pv = m.par[v];
                if (pv != NO_NODE) {   // the parent: assigned one level earlier
                    const long long j = find_label(m, v, __ldcg(m.labels + pv));
                    if (j >= 0 && __ldcg(m.H + j) <= __ldcg(m.hminp1 + v)) bk = (uint32_t)(j - (long long)m.ptr[v]);
                }
            }
            for (uint32_t q = 0; q < nb.deg && !S; ++q) {
                const uint32_t w = nb_at(m, nb, q);
                const uint32_t pw = m.pos[w];
                if (m.labels[w] != 0 && pw != NO_NODE && pw < start + i) {  // the parent: assigned one level earlier
                    const uint32_t xp = __ldcg(m.labels + w);
                    const long long j = find_label(m, v, xp);
                    if (j >= 0 && __ldcg(m.H + j) <= __ldcg(m.hminp1 + v)) bk = (uint32_t)(j - (long long)m.ptr[v]);
                    break;
                }
            }
            m.labels[v] = (uint32_t)m.view[m.ptr[v] + bk] + 1u;
            m.lidx[v] = bk;
        }
        __syncwarp();
        s = e;
    }
}


// scratch of one lane group of k_tree: h row [cap] f32 | label list [cap] u16 (only used without bitmasks) |
// label bitmask [mw] u32 | prefix popcounts [mw] u16 (padded to 4 bytes)
__host__ __device__ __forceinline__ uint32_t tree_group_bytes(uint32_t cap, uint32_t mw) { return cap * 6u + mw * 4u + ((mw * 2u + 3u) & ~3u); }

// W: weighted Potts terms (slot_weight); the unweighted instantiation is the face-graph solver.  S: a spanning forest (only
// the global-memory recursion differs: k_tree_prep<true> has classified the neighbours for the fast path)
template <int G, int MINB, bool W = false, bool S = false>
__global__ void __launch_bounds__(TREE_THREADS, MINB) k_tree(Mrf m)
{
    if (__ldcg(m.state + ST_STOP)) return;
    extern __shared__ __align__(16) unsigned char tree_dyn[];
    constexpr uint32_t NPW = 32 / G;   // nodes of one level a warp works on at a time
    constexpr int PRE = 4;             // labels of the parent a lane holds in registers ahead of the message loop
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, glane = lane & (G - 1), sub = lane / G;
    const uint32_t gmask = G == 32 ? 0xffffffffu : (((1u << (G & 31)) - 1u) << (lane & ~(uint32_t)(G - 1)));
    const uint32_t cap = m.tree_cap, mw = m.mask_words;
    // scratch of this lane group: the node's h row; its label set as a bitmask with prefix popcounts (position of a label in
    // the sorted list in O(1)); without bitmasks (more than 2047 views) the sorted list itself, searched by bisection
    unsigned char *scr = tree_dyn + ((size_t)warp * NPW + sub) * tree_group_bytes(cap, mw);
    float *Hs = reinterpret_cast<float *>(scr);
    uint16_t *Vs = reinterpret_cast<uint16_t *>(Hs + cap);
    uint32_t *Ms = reinterpret_cast<uint32_t *>(Vs + cap);
    uint16_t *Ps = reinterpret_cast<uint16_t *>(Ms + mw);
    const uint32_t nroots = m.ctl[CTL_NROOTS];
    const size_t ms = m.mstride;
    for (;;) {
        uint32_t t = 0;
        if (lane == 0) t = atomicAdd(&m.ctl[CTL_CLAIM], 1u);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= nroots) break;
        const uint4 te = __ldcg(m.ttab + t);
        const uint32_t cnt = te.x & 0x7FFFFFFFu, start = te.z;
        if (te.x >> 31) {   // a node of degree > 3 or a label list longer than the scratch
            if (lane == 0) atomicAdd(m.state + ST_SLOW, 1u);
            tree_solve_global<W, S>(m, start, cnt, lane);
            continue;
        }
        NodeRec *rec = m.rec + start;
        // ---- bottom-up: the node array is sorted by level, so walking it from its end visits the deepest level first.
        // ---- A step takes the next (up to) NPW nodes of ONE level; the records of the step after it are already on
        // ---- their way (the node array is walked in order, only the cut at a level boundary is data dependent).
        auto load_rec = [&](uint32_t hi, uint4 &r0, uint4 &r1, uint4 &r2) {   // node hi - sub, if there is one
            r0 = make_uint4(0u, 0xFFFF0000u, 0u, 0u); r1 = make_uint4(0u, 0u, 0u, 0u); r2 = r1;   // level 0xFFFF: never active
            if (hi != NO_NODE && hi >= sub) {
                const uint4 *rp = reinterpret_cast<const uint4 *>(rec + (hi - sub));
                r0 = __ldcg(rp); r1 = __ldcg(rp + 1); r2 = __ldcg(rp + 2);
            }
        };
        uint32_t hi = cnt - 1u;   // cnt >= 1: a tree has a root
        uint4 n0, n1, n2;
        load_rec(hi, n0, n1, n2);
        while (hi != NO_NODE) {
            const uint4 r0 = n0, r1 = n1, r2 = n2;
            const uint32_t i = hi - sub;   // meaningful where act
            const uint32_t lev_top = __shfl_sync(0xffffffffu, r0.y >> 16, 0);
            const bool act = hi >= sub && (r0.y >> 16) == lev_top;
            const uint32_t nact = (uint32_t)__popc(__ballot_sync(0xffffffffu, act && glane == 0));   // levels are contiguous
            hi = hi >= nact ? hi - nact : NO_NODE;
            load_rec(hi, n0, n1, n2);   // prefetch: consumed in the next step
            const uint32_t n = act ? (r0.y & 0xFFFFu) : 0u;
            const uint64_t p0 = ((uint64_t)r0.w << 32) | r0.z;
            const uint32_t e0 = r1.x, e1 = r1.y, e2 = r1.z;
            const bool c0 = (e0 & NBR_KIND) == NBR_CHILD, c1 = (e1 & NBR_KIND) == NBR_CHILD, c2 = (e2 & NBR_KIND) == NBR_CHILD;
            const uint32_t x0 = (e0 & NBR_KIND) == NBR_FIXED ? (e0 & NBR_ARG) : 0u;
            const uint32_t x1 = (e1 & NBR_KIND) == NBR_FIXED ? (e1 & NBR_ARG) : 0u;
            const uint32_t x2 = (e2 & NBR_KIND) == NBR_FIXED ? (e2 & NBR_ARG) : 0u;
            const bool has_parent = act && ((e0 & NBR_KIND) == NBR_PARENT || (e1 & NBR_KIND) == NBR_PARENT || (e2 & NBR_KIND) == NBR_PARENT);
            const uint32_t ps = r1.w & 3u, pn = has_parent ? (r1.w >> 16) : 0u;
            const uint64_t pp0 = ((uint64_t)r2.y << 32) | r2.x;
            const uint16_t *pview = m.view + pp0;
            float w0 = 1.0f, w1 = 1.0f, w2 = 1.0f;   // Potts weights of the three slots
            if constexpr (W) {
                if (act) {
                    const float *wr = m.wgt + m.adj_ptr[r0.x];
                    if (e0 & NBR_KIND) w0 = wr[0];
                    if (e1 & NBR_KIND) w1 = wr[1];
                    if (e2 & NBR_KIND) w2 = wr[2];
                }
            }
            // the parent's labels this lane will look up: loaded together with the node's own rows, not after the reduction
            uint32_t want[PRE];
#pragma unroll
            for (int q = 0; q < PRE; ++q) { const uint32_t k = glane + (uint32_t)q * G; want[q] = k < pn ? (uint32_t)pview[k] : 0u; }
            for (uint32_t w = glane; w < mw; w += G) Ms[w] = 0u;
            __syncwarp();
            const float *costv = m.cost + p0;
            const uint16_t *viewv = m.view + p0;
            const float *m0 = m.M + p0, *m1 = m.M + ms + p0, *m2 = m.M + 2 * ms + p0;
            float bh = INFINITY;
            uint32_t bk = 0xFFFFFFFFu;
#pragma unroll 2
            for (uint32_t k = glane; k < n; k += G) {
                const uint32_t vw = viewv[k];
                const uint32_t lab = vw + 1u;
                float h = costv[k];
                if (c0) h = h + __ldcg(m0 + k); else if (x0) h = h + (lab != x0 ? w0 : 0.0f);
                if (c1) h = h + __ldcg(m1 + k); else if (x1) h = h + (lab != x1 ? w1 : 0.0f);
                if (c2) h = h + __ldcg(m2 + k); else if (x2) h = h + (lab != x2 ? w2 : 0.0f);
                Hs[k] = h;
                if (mw) atomicOr(Ms + (vw >> 5), 1u << (vw & 31u)); else Vs[k] = (uint16_t)vw;
                if (h < bh) { bh = h; bk = k; }
            }
            {   // min / arg-min over the G lanes of the node by two integer warp reductions: every h is >= 0 (costs in [0, 1],
                // messages sums of such), so the unsigned order of the bit patterns is the float order; ties -> smallest index
                const uint32_t hb = __float_as_uint(bh);
                const uint32_t hmin = __reduce_min_sync(gmask, hb);
                bk = __reduce_min_sync(gmask, hb == hmin ? bk : 0xFFFFFFFFu);
                bh = __uint_as_float(hmin);
            }
            const float hm = bh + ((e0 & NBR_KIND) == NBR_PARENT ? w0 : (e1 & NBR_KIND) == NBR_PARENT ? w1 : w2);   // + weight to the parent
            __syncwarp();
            if (act && glane == 0) {   // for the top-down pass: the best label given the subtree, position and value
                rec[i].amin = bk;
                rec[i].pad = (uint32_t)viewv[bk] + 1u;
            }
            if (mw) {   // prefix popcounts of the label bitmask
                for (uint32_t w = glane; w < mw; w += G) {
                    uint32_t c = 0;
                    for (uint32_t u = 0; u < w; ++u) c += (uint32_t)__popc(Ms[u]);
                    Ps[w] = (uint16_t)c;
                }
                __syncwarp();
            }
            if (has_parent) {   // the message to the parent, one entry per label of the parent
                float *mo = m.M + (size_t)ps * ms + pp0;
                uint16_t *jo = m.J + (size_t)ps * ms + pp0;
                auto emit = [&](uint32_t k, uint32_t w) {   // w = view of the parent's label k
                    float msg = hm;
                    uint32_t jj = 0xFFFFu;
                    bool found;
                    uint32_t j;
                    if (mw) {
                        const uint32_t word = Ms[w >> 5], bit = w & 31u;
                        found = (word >> bit) & 1u;
                        j = (uint32_t)Ps[w >> 5] + (uint32_t)__popc(word & ((1u << bit) - 1u));
                    } else {
                        uint32_t lo = 0, hi2 = n;
                        while (lo < hi2) {
                            const uint32_t mid = (lo + hi2) >> 1;
                            if (Vs[mid] < w) lo = mid + 1; else hi2 = mid;
                        }
                        j = lo;
                        found = lo < n && Vs[lo] == w;
                    }
                    if (found) {
                        const float hw = Hs[j];
                        if (hw < msg) msg = hw;
                        if (hw <= hm) jj = j;
                    }
                    __stcg(mo + k, msg);
                    __stcg(jo + k, (uint16_t)jj);
                };
#pragma unroll
                for (int q = 0; q < PRE; ++q) { const uint32_t k = glane + (uint32_t)q * G; if (k < pn) emit(k, want[q]); }
                for (uint32_t k = glane + (uint32_t)PRE * G; k < pn; k += G) emit(k, (uint32_t)pview[k]);
            }
            __syncwarp();
        }
        // ---- top-down: shallowest level first, one thread per node, up to 32 nodes of one level per step ----
        for (uint32_t s = 0; s < cnt;) {
            const uint32_t i = s + lane;
            uint4 r0 = make_uint4(0u, 0xFFFF0000u, 0u, 0u), r1 = make_uint4(0u, 0u, 0u, 0u), r2 = r1;
            if (i < cnt) {
                const uint4 *rp = reinterpret_cast<const uint4 *>(rec + i);
                r0 = __ldcg(rp); r1 = __ldcg(rp + 1); r2 = __ldcg(rp + 2);
            }
            const uint32_t lev0 = __shfl_sync(0xffffffffu, r0.y >> 16, 0);
            const uint32_t same = __ballot_sync(0xffffffffu, i < cnt && (r0.y >> 16) == lev0);
            const uint32_t run = same == 0xFFFFFFFFu ? 32u : (uint32_t)__ffs((int)~same) - 1u;   // >= 1
            if (lane < run) {
                uint32_t bk = r2.z, lab = r2.w, pv = NO_NODE;
                if ((r1.x & NBR_KIND) == NBR_PARENT) pv = r1.x & NBR_ARG;
                if ((r1.y & NBR_KIND) == NBR_PARENT) pv = r1.y & NBR_ARG;
                if ((r1.z & NBR_KIND) == NBR_PARENT) pv = r1.z & NBR_ARG;
                if (pv != NO_NODE) {   // the parent was assigned one level earlier (by this warp)
                    const uint32_t ps = r1.w & 3u;
                    const uint64_t pp0 = ((uint64_t)r2.y << 32) | r2.x;
                    const uint32_t kp = __ldcg(m.lidx + pv);
                    const uint32_t plab = __ldcg(m.labels + pv);
                    const uint32_t j = __ldcg(m.J + (size_t)ps * ms + pp0 + kp);
                    if (j != 0xFFFFu) { bk = j; lab = plab; }
                }
                __stcg(m.labels + r0.x, lab);
                __stcg(m.lidx + r0.x, bk);
            }
            __syncwarp();
            s += run;
        }
    }
}

// 32.32 fixed-point energy of the owned nodes: unaries + edges counted by their lower endpoint -> efix[slot]
__global__ void __launch_bounds__(256) k_energy(Mrf m, unsigned long long *out)
{
    if (__ldcg(m.state + ST_STOP)) return;
    unsigned long long e = 0;
    for (uint32_t v = m.nb + blockIdx.x * blockDim.x + threadIdx.x; v < m.ne; v += gridDim.x * blockDim.x) {
        uint32_t x = m.labels[v];
        if (x == 0) { e += 1ull << 32; continue; }
        e += (unsigned long long)(long long)((double)m.cost[m.ptr[v] + m.lidx[v]] * 4294967296.0);
        const Nb nb = load_nb(m, v);
        for (uint32_t i = 0; i < nb.deg; ++i) {
            uint32_t w = nb_at(m, nb, i);
            uint32_t xw = m.labels[w];
            if (w > v && xw != 0 && xw != x) e += 1ull << 32;
        }
    }
    for (int s = 16; s; s >>= 1) e += __shfl_xor_sync(0xffffffffu, e, s);
    if ((threadIdx.x & 31) == 0 && e) atomicAdd(out, e);
}

// StopWhenReturnsDiminish(window, ratio) (view_selection.cpp:84), the double arithmetic of oracle/mrf.c
__global__ void k_stop(Mrf m, uint32_t t, uint32_t window, float ratio, uint32_t max_iterations)
{
    if (m.state[ST_STOP]) return;
    m.state[ST_DONE] = t;
    bool stop = t >= max_iterations;
    if (t >= window) {
        const double e0 = (double)(long long)m.efix[t - window], e1 = (double)(long long)m.efix[t];
        if (e0 <= 0.0 || (e0 - e1) / e0 < (double)ratio) stop = true;
    }
    if (stop) m.state[ST_STOP] = t;
}

// Acceptance of spanning iteration t, after k_energy and before k_restore and k_stop: fixing the non-tree neighbours at
// their old labels does not guarantee descent, so an iteration that raised the energy keeps the energy (and, through
// k_restore, the labels) of the iteration before.  One thread decides; k_restore only reads the decision.
__global__ void k_accept(Mrf m, uint32_t t)
{
    if (m.state[ST_STOP]) return;
    const long long e0 = (long long)m.efix[t - 1], e1 = (long long)m.efix[t];
    if (e1 > e0) {
        m.efix[t] = (unsigned long long)e0;
        m.ctl[CTL_REJECT] = 1u;
        m.state[ST_REJECTED] += 1u;
    }
}

__global__ void __launch_bounds__(256) k_restore(Mrf m)
{
    if (__ldcg(m.state + ST_STOP) || !__ldcg(m.ctl + CTL_REJECT)) return;
    for (uint32_t v = m.nb + blockIdx.x * blockDim.x + threadIdx.x; v < m.ne; v += gridDim.x * blockDim.x) {
        m.labels[v] = m.snap[v];
        m.lidx[v] = m.snap_lidx[v];
    }
}

// After k_accept and k_restore of a multilevel step: counts the step and its rejection, and sets CTL_KEEP unless the step
// was rejected, so that only a rejected step projects the restored coarse labels onto the faces again
__global__ void k_step_count(Mrf m)
{
    const bool stopped = m.state[ST_STOP] != 0u, rejected = m.ctl[CTL_REJECT] != 0u;
    m.ctl[CTL_KEEP] = stopped || !rejected ? 1u : 0u;
    if (stopped) return;
    m.state[ST_STEPS] += 1u;
    if (rejected) m.state[ST_STEP_REJ] += 1u;
}

// label range check + unseen count (view_selection.cpp:121-132)
__global__ void __launch_bounds__(256) k_label_check(Mrf m)
{
    uint32_t bad = 0, unseen = 0;
    for (uint32_t v = m.nb + blockIdx.x * blockDim.x + threadIdx.x; v < m.ne; v += gridDim.x * blockDim.x) {
        const uint32_t x = m.labels[v];
        if (m.K && x > m.K) ++bad;
        if (x == 0) ++unseen;
    }
    for (int s = 16; s; s >>= 1) { bad += __shfl_xor_sync(0xffffffffu, bad, s); unseen += __shfl_xor_sync(0xffffffffu, unseen, s); }
    if ((threadIdx.x & 31) == 0) {
        if (bad) atomicAdd(m.state + ST_BAD, bad);
        if (unseen) atomicAdd(m.state + ST_UNSEEN, unseen);
    }
}


// ---- multi-GPU (one process per GPU): boundary-label halo + energy all-reduce through NVLink peer memory -----------
// Rank r owns the faces [r * part_size, (r + 1) * part_size) and holds a full-length label array inside a block its
// peers have mapped (cudaIpc).  After every sweep a rank STORES the labels of its boundary faces -- the faces with a
// neighbour on another rank, O(sqrt(F / P)) per cut (view_selection.cpp:29-42 couples faces only across an edge) --
// straight into the label arrays of exactly the ranks that own such a neighbour, then all ranks meet at an epoch-flag
// barrier in peer memory.  The energy for the stop rule goes the same way: every rank stores its fixed-point partial into
// slot [t][rank] of every peer, meets, and adds the slots in rank order, so all ranks take the identical decision from
// identical integers without a host round trip or an NCCL call.
constexpr int MRF_MAX_RANKS = 8;
constexpr uint32_t MRF_SLOTS = 1026;   // iterations 0 .. max_iterations (<= 1022) + scratch
struct MrfPeers {
    uint32_t rank, nranks;
    uint32_t *labels[MRF_MAX_RANKS];            // every rank's full-length label array
    unsigned long long *eslot[MRF_MAX_RANKS];   // [MRF_SLOTS][MRF_MAX_RANKS] partial energies, per rank
    uint32_t *flag[MRF_MAX_RANKS];              // [MRF_MAX_RANKS] barrier epochs, per rank
    unsigned long long spin_limit;
};
__host__ __device__ inline size_t mrf_align256(size_t n) { return (n + 255) & ~(size_t)255; }
__host__ __device__ inline size_t mrf_block_bytes(uint32_t F)
{
    return mrf_align256((size_t)F * 4) + mrf_align256((size_t)MRF_SLOTS * MRF_MAX_RANKS * 8) + 256;
}

// ---- system-scope flag primitives (the host emulation replaces this block) ----
__device__ __forceinline__ void st_release_sys(uint32_t *p, uint32_t v)
{
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t *p)
{
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// ---- end of flag primitives ----

// boundary faces of the owned range and the ranks each of them has a neighbour on
__global__ void __launch_bounds__(256) k_halo_build(Mrf m, uint32_t *cnt, uint32_t *list, uint32_t *lmask)
{
    const uint32_t v = m.nb + blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= m.ne) return;
    const Nb nb = load_nb(m, v);
    uint32_t mask = 0;
    for (uint32_t i = 0; i < nb.deg; ++i) {
        const uint32_t w = nb_at(m, nb, i);
        if (!owned(m, w)) mask |= 1u << (w / m.part_size);
    }
    if (mask) {
        const uint32_t i = atomicAdd(cnt, 1u);
        list[i] = v;
        lmask[i] = mask;
    }
}

__global__ void __launch_bounds__(256) k_halo_push(Mrf m, MrfPeers pr, const uint32_t *__restrict__ list,
                                                   const uint32_t *__restrict__ lmask, const uint32_t *__restrict__ cnt)
{
    if (__ldcg(m.state + ST_STOP)) return;
    const uint32_t n = *cnt;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t v = list[i], x = m.labels[v];
        for (uint32_t mk = lmask[i]; mk; mk &= mk - 1u) {
            const uint32_t k = (uint32_t)__ffs((int)mk) - 1u;
            if (k < pr.nranks && k != pr.rank) pr.labels[k][v] = x;
        }
    }
    __threadfence_system();
}

// after the last iteration: every rank gets every label (the seam assembly that follows is replicated)
__global__ void __launch_bounds__(256) k_range_push(Mrf m, MrfPeers pr)
{
    for (uint32_t v = m.nb + blockIdx.x * blockDim.x + threadIdx.x; v < m.ne; v += gridDim.x * blockDim.x) {
        const uint32_t x = m.labels[v];
        for (uint32_t k = 0; k < pr.nranks; ++k)
            if (k != pr.rank) pr.labels[k][v] = x;
    }
    __threadfence_system();
}

// One warp.  phase 0: all ranks meet (every label pushed before is visible afterwards).  phase 1: additionally the
// partial energies elocal[t] are all-reduced into m.efix[t] (rank order) and the stop rule of iteration t is applied.
// phase 2: barrier that also runs after the stop rule has fired (the final label all-gather).
__global__ void k_mg_sync(Mrf m, MrfPeers pr, uint32_t epoch, int phase, uint32_t t, uint32_t window, float ratio,
                          uint32_t max_iterations, const unsigned long long *elocal)
{
    if (phase != 2 && __ldcg(m.state + ST_STOP)) return;
    const uint32_t k = threadIdx.x;
    if (k < pr.nranks) {
        if (phase == 1) {
            pr.eslot[k][(size_t)t * MRF_MAX_RANKS + pr.rank] = elocal[t];
            __threadfence_system();
        }
        st_release_sys(pr.flag[k] + pr.rank, epoch);
        unsigned long long spins = 0;
        while ((int32_t)(ld_acquire_sys(pr.flag[pr.rank] + k) - epoch) < 0) {
            __nanosleep(64);
            if (++spins > pr.spin_limit) { atomicAdd(m.state + ST_ERR, 1u); break; }
        }
    }
    __syncwarp();
    if (k != 0) return;
    if (__ldcg(m.state + ST_ERR)) { if (!m.state[ST_STOP]) m.state[ST_STOP] = t ? t : 1u; return; }   // a peer is gone: halt what is queued
    if (phase != 1) return;
    unsigned long long sum = 0;
    for (uint32_t r = 0; r < pr.nranks; ++r) sum += __ldcg(pr.eslot[pr.rank] + (size_t)t * MRF_MAX_RANKS + r);
    m.efix[t] = sum;
    if (t == 0) return;
    m.state[ST_DONE] = t;
    bool stop = t >= max_iterations;
    if (t >= window) {
        const double e0 = (double)(long long)m.efix[t - window], e1 = (double)(long long)sum;
        if (e0 <= 0.0 || (e0 - e1) / e0 < (double)ratio) stop = true;
    }
    if (stop) m.state[ST_STOP] = t;
}

}  // namespace

struct MrfMgState {
    void *block = nullptr;                      // own peer-visible block (cudaMalloc)
    void *peer[MRF_MAX_RANKS] = {nullptr};      // opened peers (peer[rank] = block)
    bool opened[MRF_MAX_RANKS] = {false};
    uint32_t F = 0, rank = 0, nranks = 1, epoch = 0;
    DevBuf<uint32_t> halo_list, halo_mask, halo_cnt;
    DevBuf<unsigned long long> elocal;         // [MRF_SLOTS] partial energies of this rank
};

namespace {

Mrf make_mrf(b2tex_ctx *c, uint32_t iter)
{
    Mrf m;
    m.F = c->F; m.nb = c->face_begin; m.ne = c->face_end;
    m.adj_ptr = c->adj_ptr.p; m.adj_idx = c->adj_idx.p;
    m.adj4 = c->mrf_adj4.p;
    m.ptr = c->dc_ptr.p; m.view = c->dc_view.p; m.cost = c->dc_cost.p;
    m.H = c->mrf_H.p; m.hminp1 = c->mrf_hminp1.p; m.amin = c->mrf_amin.p; m.level = c->mrf_level.p;
    m.labels = c->labels.p; m.lidx = c->mrf_lidx.p;
    m.order = c->mrf_order.p; m.olev = c->mrf_olev.p; m.pos = c->mrf_pos.p;
    m.tjoin = c->mrf_tjoin.p; m.ttab = c->mrf_ttab.p;
    m.ctl = c->mrf_ctl.p; m.state = c->mrf_state.p;
    m.queue = c->mrf_queue.p; m.qstamp = c->mrf_queue.p + 2 * (size_t)c->F;
    m.efix = c->mrf_energy.p;
    m.dbg = c->mrf_dbg.n ? c->mrf_dbg.p : nullptr;
    m.K = c->K;
    m.mask_words = c->mrf_mask_words;
    const b2tex_mrf_params &p = c->mrf_params;
    uint32_t P = p.num_parts ? p.num_parts : 1;
    m.part_size = (c->F + P - 1) / P; if (!m.part_size) m.part_size = 1;
    m.rounds = p.rounds;
    if (p.root_div == 0) m.rdiv = 0;
    else { uint32_t cap = c->F / 8u; if (cap < 1u) cap = 1u; m.rdiv = p.root_div < cap ? p.root_div : cap; }
    m.seed = p.seed;
    m.iter = iter;
    m.tree_smem = c->mrf_tree_smem;
    m.rec = reinterpret_cast<NodeRec *>(c->mrf_rec.p);
    m.M = c->mrf_M.p; m.J = c->mrf_J.p; m.mstride = c->nnz;
    m.tree_cap = c->mrf_tree_cap;
    m.wgt = nullptr;
    m.par = c->mrf_par.p;
    m.snap = c->mrf_snap.p; m.snap_lidx = c->mrf_snap.p ? c->mrf_snap.p + c->F : nullptr;
    return m;
}

// The contracted MRF of mrf_contract (single GPU, whole mesh) with the fine run's scratch, seed and iteration numbers.  The
// push stamps stay where make_mrf put them (queue + 2 F, beyond both frontier lists of the n <= F coarse nodes): a stamp is
// unique per (iteration, round), and iteration numbers go on from the fine phases.
Mrf make_coarse_mrf(b2tex_ctx *c, uint32_t iter)
{
    Mrf m = make_mrf(c, iter);
    const uint32_t n = c->ml_nodes;
    m.F = n; m.nb = 0; m.ne = n;
    m.adj_ptr = c->ml_cadj_ptr.p; m.adj_idx = c->ml_cadj_idx.p; m.adj4 = c->ml_cadj4.p; m.wgt = c->ml_cwgt.p;
    m.ptr = c->ml_cptr.p; m.view = c->ml_cview.p; m.cost = c->ml_ccost.p;
    m.labels = c->ml_clabels.p; m.lidx = c->ml_clidx.p;
    m.part_size = n ? n : 1;
    const uint32_t rd = c->mrf_params.root_div;
    if (rd == 0) m.rdiv = 0;
    else { uint32_t cap = n / 8u; if (cap < 1u) cap = 1u; m.rdiv = rd < cap ? rd : cap; }
    return m;
}

template <typename K>
int coop_grid(b2tex_ctx *c, K kernel, size_t smem, int *grid, int threads = 256)
{
    int per_sm = 0;
    B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem));
    if (per_sm < 1) { set_error("mrf kernel cannot be resident"); return B2TEX_ERR_CUDA; }
    *grid = c->num_sms * per_sm;
    return B2TEX_OK;
}

template <bool S = false>
int launch_forest(b2tex_ctx *c, Mrf &m, int build_trees)
{
    cudaStream_t s = c->stream;
    int grid = 0;
    // few fat blocks: the cost of grid.sync() grows with the number of blocks
    B2_TRY(coop_grid(c, k_forest<S>, 0, &grid, FOREST_THREADS));
    if (grid > c->num_sms) grid = c->num_sms;  // one fat block per SM: cheapest grid.sync()
    if (const char *e = getenv("B2TEX_FOREST_BLOCKS_PER_SM")) grid = c->num_sms * std::max(1, atoi(e));
    uint32_t n = m.ne - m.nb;
    int need = (int)((n + FOREST_THREADS - 1) / FOREST_THREADS);
    if (grid > need) grid = need > 0 ? need : 1;
    B2_CUDA(cudaMemsetAsync(m.ctl, 0, CTL_WORDS * sizeof(uint32_t), s));
    void *args[] = {&m, &build_trees};
    count_launch();
    B2_CUDA(cudaLaunchCooperativeKernel((void *)k_forest<S>, dim3(grid), dim3(FOREST_THREADS), args, 0, s));
    return B2TEX_OK;
}

template <int G, int MINB, bool W, bool S>
int launch_tree_variant(b2tex_ctx *c, Mrf &m)
{
    static bool attr_set = false;   // opt in to > 48 KB of dynamic shared memory (per function, once)
    if (!attr_set) {
        B2_CUDA(cudaFuncSetAttribute(k_tree<G, MINB, W, S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TREE_SMEM_MAX));
        attr_set = true;
    }
    int per_sm = 0;
    B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_tree<G, MINB, W, S>, TREE_THREADS, m.tree_smem));
    if (per_sm < 1) { set_error("k_tree cannot be resident with %u bytes of shared memory", m.tree_smem); return B2TEX_ERR_CUDA; }
    const int grid = c->num_sms * per_sm;
    B2_LAUNCH k_tree<G, MINB, W, S><<<grid, TREE_THREADS, m.tree_smem, c->stream>>>(m);
    B2_KERNEL_CHECK();
    return B2TEX_OK;
}

template <int G, bool W = false, bool S = false>
int launch_tree(b2tex_ctx *c, Mrf &m)
{
    const uint32_t n = m.ne - m.nb;
    B2_LAUNCH k_tree_prep<S><<<(n + 255) / 256, 256, 0, c->stream>>>(m);   // at most n forest nodes; the kernel reads the count
    // 2 CTAs of 512 threads per SM (64 registers) or 3 (40 registers, a few spills): the kernel lives on resident warps, but
    // on an H100 SXM (700 W) the spill-free variant is faster (C3: k_tree 28.7 against 44.6 ms per pass)
    static const int minb = getenv("B2TEX_TREE_BLOCKS") ? atoi(getenv("B2TEX_TREE_BLOCKS")) : 2;
    return minb == 3 ? launch_tree_variant<G, 3, W, S>(c, m) : launch_tree_variant<G, 2, W, S>(c, m);
}

// peers of this context, or nranks == 1
MrfPeers make_peers(b2tex_ctx *c)
{
    MrfPeers pr;
    memset(&pr, 0, sizeof(pr));
    pr.nranks = 1;
    MrfMgState *g = c->mrf_mg;
    if (!g || g->nranks < 2) return pr;
    pr.rank = g->rank; pr.nranks = g->nranks;
    for (uint32_t k = 0; k < g->nranks; ++k) {
        char *b = (char *)g->peer[k];
        pr.labels[k] = (uint32_t *)b;
        pr.eslot[k] = (unsigned long long *)(b + mrf_align256((size_t)g->F * 4));
        pr.flag[k] = (uint32_t *)(b + mrf_align256((size_t)g->F * 4) + mrf_align256((size_t)MRF_SLOTS * MRF_MAX_RANKS * 8));
    }
    pr.spin_limit = 40ull * 1000 * 1000;   // x (64 ns sleep + a system-scope load): several seconds
    return pr;
}
bool mg_active(b2tex_ctx *c) { return c->mrf_mg && c->mrf_mg->nranks > 1; }
// epoch of the barrier of iteration t (0 = init), phase 0 (labels) / 1 (energy); 1 = entry barrier of the run
uint32_t mg_epoch(b2tex_ctx *c, uint32_t t, int phase) { return c->mrf_mg->epoch + 2u + 2u * t + (uint32_t)phase; }

int launch_energy(b2tex_ctx *c, Mrf &m, uint32_t t)
{
    unsigned long long *out = mg_active(c) ? c->mrf_mg->elocal.p + t : m.efix + t;
    B2_LAUNCH k_energy<<<std::max(1, c->num_sms * 8), 256, 0, c->stream>>>(m, out);
    B2_KERNEL_CHECK();
    return B2TEX_OK;
}

// k_stop on the phase's own iteration numbers (single GPU): ST_STOP / ST_DONE are relative to t_ref
void enqueue_stop(b2tex_ctx *c, const Mrf &m, uint32_t t, uint32_t t_ref)
{
    const b2tex_mrf_params &p = c->mrf_params;
    Mrf ms = m;
    ms.efix = m.efix + t_ref;
    B2_LAUNCH k_stop<<<1, 1, 0, c->stream>>>(ms, t - t_ref, p.window ? p.window : 1u, p.ratio, p.max_iterations - t_ref);
}

// label halo -> barrier -> partial energies -> barrier + all-reduce + stop rule (multi-GPU), or energy + stop rule.
// t_ref: the iteration the stop rule's window restarts from (a phase of multilevel or spanning-tree view selection, single
// GPU only).  accept: a spanning iteration, undone if it raised the energy (single GPU only).
int enqueue_exchange_and_energy(b2tex_ctx *c, Mrf &m, uint32_t t, bool stop_rule, uint32_t t_ref = 0, bool accept = false)
{
    cudaStream_t s = c->stream;
    const b2tex_mrf_params &p = c->mrf_params;
    const uint32_t window = p.window ? p.window : 1u;
    if (!mg_active(c)) {
        {
            ScopedTimer te(c, "mrf.k_energy", 12.0 * (double)(m.ne - m.nb));
            B2_TRY(launch_energy(c, m, t));
        }
        if (accept) {
            ScopedTimer ta(c, "mrf.accept");
            B2_LAUNCH k_accept<<<1, 1, 0, s>>>(m, t);
            B2_LAUNCH k_restore<<<std::max(1, c->num_sms * 8), 256, 0, s>>>(m);
        }
        if (stop_rule) enqueue_stop(c, m, t, t_ref);
        B2_KERNEL_CHECK();
        return B2TEX_OK;
    }
    MrfMgState *g = c->mrf_mg;
    MrfPeers pr = make_peers(c);
    {
        ScopedTimer th(c, "mrf.halo_exchange");
        B2_LAUNCH k_halo_push<<<std::max(1, c->num_sms), 256, 0, s>>>(m, pr, g->halo_list.p, g->halo_mask.p, g->halo_cnt.p);
        B2_LAUNCH k_mg_sync<<<1, 32, 0, s>>>(m, pr, mg_epoch(c, t, 0), 0, t, window, p.ratio, p.max_iterations, g->elocal.p);
    }
    {
        ScopedTimer te(c, "mrf.k_energy", 12.0 * (double)(m.ne - m.nb));
        B2_TRY(launch_energy(c, m, t));
    }
    ScopedTimer ta(c, "mrf.energy_allreduce");
    B2_LAUNCH k_mg_sync<<<1, 32, 0, s>>>(m, pr, mg_epoch(c, t, 1), 1, t, stop_rule ? window : 0xFFFFFFFFu, p.ratio,
                                 stop_rule ? p.max_iterations : 0xFFFFFFFFu, g->elocal.p);
    B2_KERNEL_CHECK();
    return B2TEX_OK;
}

int enqueue_iteration(b2tex_ctx *c, Mrf &m, bool stop_rule, uint32_t t_ref = 0)
{
    if (m.ne <= m.nb && !mg_active(c)) return B2TEX_OK;
    {
        ScopedTimer tf(c, "mrf.k_forest", 20.0 * (double)(m.ne - m.nb));
        B2_TRY(launch_forest(c, m, 1));
    }
    {
        ScopedTimer tu(c, "mrf.k_tree");   // bytes are filled in after the run (forest coverage is known then)
        switch (c->mrf_group) {
            case 4: B2_TRY(launch_tree<4>(c, m)); break;
            case 8: B2_TRY(launch_tree<8>(c, m)); break;
            case 16: B2_TRY(launch_tree<16>(c, m)); break;
            default: B2_TRY(launch_tree<32>(c, m)); break;
        }
    }
    return enqueue_exchange_and_energy(c, m, m.iter, stop_rule, t_ref);
}

// one iteration on the spanning forest (single GPU, whole mesh), accepted or undone, and the stop rule (window from t_ref)
int enqueue_spanning_iteration(b2tex_ctx *c, Mrf &m, uint32_t t_ref)
{
    {
        ScopedTimer tf(c, "mrf.k_forest_spanning");
        B2_TRY(launch_forest<true>(c, m, 1));
    }
    {
        ScopedTimer tu(c, "mrf.k_tree_spanning");
        switch (c->mrf_group) {
            case 4: B2_TRY((launch_tree<4, false, true>(c, m))); break;
            case 8: B2_TRY((launch_tree<8, false, true>(c, m))); break;
            case 16: B2_TRY((launch_tree<16, false, true>(c, m))); break;
            default: B2_TRY((launch_tree<32, false, true>(c, m))); break;
        }
    }
    return enqueue_exchange_and_energy(c, m, m.iter, true, t_ref, true);
}

// one iteration of the BCD on the contracted MRF (weighted Potts terms), the projection onto the faces, and the fine
// energy + stop rule (window restarted at t_ref)
int enqueue_coarse_iteration(b2tex_ctx *c, uint32_t t, uint32_t t_ref)
{
    Mrf cm = make_coarse_mrf(c, t);
    {
        ScopedTimer tf(c, "mrf.k_forest");
        B2_TRY(launch_forest(c, cm, 1));
    }
    {
        ScopedTimer tu(c, "mrf.k_tree_weighted");
        switch (c->mrf_group) {
            case 4: B2_TRY((launch_tree<4, true>(c, cm))); break;
            case 8: B2_TRY((launch_tree<8, true>(c, cm))); break;
            case 16: B2_TRY((launch_tree<16, true>(c, cm))); break;
            default: B2_TRY((launch_tree<32, true>(c, cm))); break;
        }
    }
    Mrf m = make_mrf(c, t);
    {
        ScopedTimer tp(c, "mrf_ml.project");
        B2_TRY(mrf_project(c, m.state + ST_STOP));
    }
    return enqueue_exchange_and_energy(c, m, t, true, t_ref);
}

// One multilevel step of the spanning phase (oracle/mrf_mapmap.c) as iteration t: contract the labels, one spanning-tree
// iteration with weighted Potts terms on the contracted MRF, the projection, the fine energy and its acceptance, and the
// stop rule (window from t_ref).  A rejected step restores the coarse labels and positions from the snapshot k_forest<true>
// took and projects them again: every face gets the label of its region, which is the label it had when it was contracted,
// so no snapshot of the faces is needed.  The contraction reads its sizes back; everything after it is queued.
int enqueue_multilevel_step(b2tex_ctx *c, uint32_t t, uint32_t t_ref, uint32_t *num_nodes)
{
    cudaStream_t s = c->stream;
    {
        ScopedTimer tc(c, "mrf_ml.contract");
        B2_TRY(mrf_contract(c, num_nodes));
        if (*num_nodes) B2_LAUNCH k_build_adj4<<<(*num_nodes + 255) / 256, 256, 0, s>>>(*num_nodes, c->ml_cadj_ptr.p, c->ml_cadj_idx.p, c->ml_cadj4.p);
        B2_KERNEL_CHECK();
    }
    if (!*num_nodes) { set_error("multilevel step: the contraction has no nodes"); return B2TEX_ERR_ARG; }
    Mrf cm = make_coarse_mrf(c, t);
    {
        ScopedTimer tf(c, "mrf.k_forest_spanning");
        B2_TRY(launch_forest<true>(c, cm, 1));
    }
    {
        ScopedTimer tu(c, "mrf.k_tree_spanning_weighted");
        switch (c->mrf_group) {
            case 4: B2_TRY((launch_tree<4, true, true>(c, cm))); break;
            case 8: B2_TRY((launch_tree<8, true, true>(c, cm))); break;
            case 16: B2_TRY((launch_tree<16, true, true>(c, cm))); break;
            default: B2_TRY((launch_tree<32, true, true>(c, cm))); break;
        }
    }
    Mrf m = make_mrf(c, t);
    {
        ScopedTimer tp(c, "mrf_ml.project");
        B2_TRY(mrf_project(c, m.state + ST_STOP));
    }
    {
        ScopedTimer te(c, "mrf.k_energy", 12.0 * (double)(m.ne - m.nb));
        B2_TRY(launch_energy(c, m, t));
    }
    {
        ScopedTimer ta(c, "mrf.accept");
        B2_LAUNCH k_accept<<<1, 1, 0, s>>>(m, t);
        B2_LAUNCH k_restore<<<std::max(1, c->num_sms * 8), 256, 0, s>>>(cm);
        B2_LAUNCH k_step_count<<<1, 1, 0, s>>>(m);
        B2_KERNEL_CHECK();
        B2_TRY(mrf_project(c, m.ctl + CTL_KEEP));
    }
    enqueue_stop(c, m, t, t_ref);
    B2_KERNEL_CHECK();
    return B2TEX_OK;
}

int alloc_mrf(b2tex_ctx *c, const b2tex_mrf_params *p)
{
    B2_TRY(require(c, COSTS | ADJ, "view selection"));
    if (p->rounds + 2 > (uint32_t)MAX_LEVELS) { set_error("mrf rounds too large"); return B2TEX_ERR_ARG; }
    if (p->max_iterations + 4 > MRF_SLOTS) { set_error("view selection: at most %u iterations", MRF_SLOTS - 4); return B2TEX_ERR_ARG; }
    c->mrf_params = *p;
    const size_t F = c->F;
    if (mg_active(c)) {
        MrfMgState *g = c->mrf_mg;
        const uint32_t P = g->nranks, psz = (uint32_t)((F + P - 1) / P);
        if (g->F != F || (p->num_parts ? p->num_parts : 1) != P || c->face_begin != std::min<size_t>(F, (size_t)g->rank * psz) ||
            c->face_end != std::min<size_t>(F, (size_t)(g->rank + 1) * psz)) {
            set_error("multi-GPU view selection: the face range must be [rank * ceil(F / P), (rank + 1) * ceil(F / P)) and "
                      "num_parts = P (F %zu, P %u, range %u..%u, num_parts %u)", F, P, c->face_begin, c->face_end, p->num_parts);
            return B2TEX_ERR_ARG;
        }
        for (uint32_t k = 0; k < P; ++k)
            if (!g->peer[k]) { set_error("multi-GPU view selection: peer %u not imported", k); return B2TEX_ERR_ARG; }
        const size_t n = c->face_end - c->face_begin;
        B2_TRY(g->elocal.alloc(MRF_SLOTS));
        B2_TRY(g->halo_list.alloc(n)); B2_TRY(g->halo_mask.alloc(n)); B2_TRY(g->halo_cnt.alloc(1));
    }
    // pinned: [0, 64) stop flags the host polls, then a read-back area (a cudaMemcpyAsync to PAGEABLE memory waits for the
    // stream inside the driver; with several ranks driven from one process that blocks the peers' launches)
    if (!c->mrf_host_flags) B2_CUDA(cudaHostAlloc((void **)&c->mrf_host_flags, (64 + 2 * MRF_SLOTS + 64) * sizeof(uint32_t), cudaHostAllocDefault));
    B2_TRY(c->mrf_H.alloc(c->nnz));
    B2_TRY(c->mrf_M.alloc(3 * (size_t)c->nnz));
    B2_TRY(c->mrf_J.alloc(3 * (size_t)c->nnz));
    B2_TRY(c->mrf_rec.alloc(3 * F));   // 48-byte records as uint4 triples
    B2_TRY(c->mrf_hminp1.alloc(F));
    B2_TRY(c->mrf_amin.alloc(F));
    B2_TRY(c->mrf_level.alloc(F));
    B2_TRY(c->mrf_lidx.alloc(F));
    B2_TRY(c->mrf_order.alloc(F));
    B2_TRY(c->mrf_olev.alloc(F));
    B2_TRY(c->mrf_pos.alloc(F));
    B2_CUDA(cudaMemsetAsync(c->mrf_pos.p, 0xFF, F * sizeof(uint32_t), c->stream));  // nodes of other ranks never enter a tree
    B2_TRY(c->mrf_tjoin.alloc(F));
    B2_TRY(c->mrf_ttab.alloc(F));
    B2_TRY(c->mrf_queue.alloc(3 * F));   // frontier lists [2][F] | qstamp [F]
    B2_TRY(c->mrf_queue.zero(c->stream));
    B2_TRY(c->mrf_ctl.alloc(CTL_WORDS));
    B2_TRY(c->mrf_state.alloc(ST_WORDS));
    B2_TRY(c->mrf_state.zero(c->stream));
    B2_TRY(c->mrf_energy.alloc(MRF_SLOTS));
    B2_TRY(c->mrf_energy.zero(c->stream));
    static const bool forest_timing = getenv("B2TEX_FOREST_TIMING") != nullptr;
    if (forest_timing) { B2_TRY(c->mrf_dbg.alloc(16)); B2_TRY(c->mrf_dbg.zero(c->stream)); }
    if (p->use_spanning_tree) {   // parents, and the labels and label positions at the start of an iteration
        B2_TRY(c->mrf_par.alloc(F));
        B2_TRY(c->mrf_snap.alloc(2 * F));
    }
    B2_TRY(c->mrf_adj4.alloc(F));
    if (F) B2_LAUNCH k_build_adj4<<<(unsigned)((F + 255) / 256), 256, 0, c->stream>>>((uint32_t)F, c->adj_ptr.p, c->adj_idx.p, c->mrf_adj4.p);
    if (!(c->valid & LABELS) || c->labels.n != F) { B2_TRY(c->labels.alloc(F)); B2_TRY(c->labels.zero(c->stream)); }
    uint32_t nodes = c->face_end - c->face_begin;
    double rho = nodes ? (double)c->nnz / nodes : 0.0;
    // lanes per node: a level of one tree holds only a few nodes, so wide groups idle on short label lists
    c->mrf_group = rho >= 64 ? 32 : rho >= 12 ? 16 : rho >= 6 ? 8 : 4;
    // fewer trees than resident warps (small meshes, or one rank of many): a launch lasts as long as its largest tree, and
    // half as many lanes per node mean twice as many nodes of a level per step
    if (c->mrf_group == 16 && (uint64_t)nodes / std::max(1u, p->root_div ? p->root_div : 1u) < (uint64_t)c->num_sms * 32u) c->mrf_group = 8;
    if (const char *g = getenv("B2TEX_MRF_GROUP")) {
        int v = atoi(g);
        if (v == 4 || v == 8 || v == 16 || v == 32) c->mrf_group = v;
    }
    // label bitmasks: labels are view+1 <= K
    uint32_t words = (c->K + 1 + 31) / 32;
    static const bool no_masks = getenv("B2TEX_NO_MASKS") != nullptr;
    c->mrf_mask_words = (c->K == 0 || words > (uint32_t)MAX_MASK_WORDS || no_masks) ? 0 : words;
    // shared-memory scratch of k_tree: one h row + label list (6 bytes per label) per lane group; the longest label
    // list decides, up to 1024 labels and as long as the scratch of all lane groups fits TREE_SMEM_MAX (trees with a
    // longer list go through the global tables)
    uint32_t maxn = 0;
    if (nodes) {
        B2_TRY(c->s_limits.alloc(1));
        B2_TRY(c->s_limits.zero(c->stream));
        B2_LAUNCH k_max_labels<<<std::max(1, c->num_sms * 4), 256, 0, c->stream>>>(c->dc_ptr.p, c->face_begin, c->face_end, c->s_limits.p);
        B2_KERNEL_CHECK();
        B2_CUDA(cudaMemcpyAsync(c->mrf_host_flags + 32, c->s_limits.p, 4, cudaMemcpyDeviceToHost, c->stream));
        B2_CUDA(cudaStreamSynchronize(c->stream));
        maxn = c->mrf_host_flags[32];
    }
    uint32_t cap = std::min(1024u, std::max(16u, (maxn + 15u) & ~15u));
    if (const char *e = getenv("B2TEX_TREE_CAP")) cap = (uint32_t)std::max(16, std::min(1024, atoi(e) & ~15));
    const uint32_t groups = (uint32_t)TREE_WARPS * (32u / (uint32_t)c->mrf_group);
    while (cap > 16u && groups * tree_group_bytes(cap, c->mrf_mask_words) > TREE_SMEM_MAX) cap -= 16u;
    c->mrf_tree_cap = cap;
    c->mrf_tree_smem = groups * tree_group_bytes(cap, c->mrf_mask_words);
    return B2TEX_OK;
}

int read_energy(b2tex_ctx *c, const Mrf &m, uint32_t slot, int64_t *efix)
{
    unsigned long long *pin = reinterpret_cast<unsigned long long *>(c->mrf_host_flags + 64);
    B2_CUDA(cudaMemcpyAsync(pin, m.efix + slot, sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    *efix = (int64_t)pin[0];
    return B2TEX_OK;
}

}  // namespace

// init: arg-min labels of the owned faces, (multi-GPU: boundary labels to the peers,) energy of the initial labeling
int mrf_init(b2tex_ctx *c, const b2tex_mrf_params *p, int64_t *efix)
{
    invalidate(c, MRF);
    B2_TRY(alloc_mrf(c, p));   // keeps the labels of faces outside the owned range while they are valid
    invalidate(c, LABELS);
    Mrf m = make_mrf(c, 0);
    cudaStream_t s = c->stream;
    const int grid = std::max(1, c->num_sms * 8);
    if (mg_active(c)) {
        MrfMgState *g = c->mrf_mg;
        MrfPeers pr = make_peers(c);
        B2_TRY(g->elocal.zero(s));
        const uint32_t n = m.ne - m.nb;
        B2_TRY(g->halo_cnt.zero(s));
        if (n) B2_LAUNCH k_halo_build<<<(n + 255) / 256, 256, 0, s>>>(m, g->halo_cnt.p, g->halo_list.p, g->halo_mask.p);
        // entry barrier: every rank is done with the labels of the previous run before anybody overwrites them
        B2_LAUNCH k_mg_sync<<<1, 32, 0, s>>>(m, pr, g->epoch + 1u, 0, 0u, 1u, 0.0f, 0xFFFFFFFFu, g->elocal.p);
        B2_KERNEL_CHECK();
    }
    if (m.ne > m.nb) {
        ScopedTimer tm(c, "mrf_init");
        switch (c->mrf_group) {
            case 4: B2_LAUNCH k_init_labels<4><<<grid, 256, 0, s>>>(m); break;
            case 8: B2_LAUNCH k_init_labels<8><<<grid, 256, 0, s>>>(m); break;
            case 16: B2_LAUNCH k_init_labels<16><<<grid, 256, 0, s>>>(m); break;
            default: B2_LAUNCH k_init_labels<32><<<grid, 256, 0, s>>>(m); break;
        }
        B2_KERNEL_CHECK();
    }
    if (m.ne > m.nb || mg_active(c)) B2_TRY(enqueue_exchange_and_energy(c, m, 0u, false));
    B2_TRY(read_energy(c, m, 0u, efix));
    mark_valid(c, LABELS | MRF);
    return B2TEX_OK;
}

// every allocation of a run, nothing else: a caller that drives several ranks from ONE process (threads) prepares all of
// them before the first rank starts, because cudaMalloc waits for the whole device and a rank that already spins in a
// cross-rank barrier kernel would never be released (separate processes / devices do not have that problem)
int mrf_prepare(b2tex_ctx *c, const b2tex_mrf_params *p)
{
    B2_TRY(alloc_mrf(c, p));
    // ... and every kernel of the run is loaded now: with lazy module loading the FIRST launch of a kernel synchronises
    // the context, which would also wait for a peer rank's spinning barrier kernel
    cudaFuncAttributes fa;
    const void *fns[] = {(const void *)k_forest<false>, (const void *)k_energy, (const void *)k_stop, (const void *)k_label_check,
                         (const void *)k_build_adj4, (const void *)k_halo_build, (const void *)k_halo_push, (const void *)k_range_push,
                         (const void *)k_mg_sync, (const void *)k_tree_prep<false>, (const void *)k_max_labels, (const void *)k_tree<4, 3>, (const void *)k_tree<8, 3>, (const void *)k_tree<16, 3>,
                         (const void *)k_tree<32, 3>, (const void *)k_tree<4, 2>, (const void *)k_tree<8, 2>, (const void *)k_tree<16, 2>,
                         (const void *)k_tree<32, 2>, (const void *)k_init_labels<4>, (const void *)k_init_labels<8>,
                         (const void *)k_init_labels<16>, (const void *)k_init_labels<32>};
    for (const void *f : fns) B2_CUDA(cudaFuncGetAttributes(&fa, f));
    return B2TEX_OK;
}

// one iteration, energy read back (single GPU, or the building block of a host-driven sharded loop over NCCL)
int mrf_iterate(b2tex_ctx *c, uint32_t t, int64_t *efix)
{
    B2_TRY(require(c, MRF, "mrf_iterate"));
    if (t == 0 || t > c->mrf_params.max_iterations) { set_error("mrf_iterate: iterations are numbered from 1 to max_iterations"); return B2TEX_ERR_ARG; }
    invalidate(c, LABELS);
    Mrf m = make_mrf(c, t);
    B2_CUDA(cudaMemsetAsync(m.efix + t, 0, sizeof(unsigned long long), c->stream));
    if (mg_active(c)) B2_CUDA(cudaMemsetAsync(c->mrf_mg->elocal.p + t, 0, sizeof(unsigned long long), c->stream));
    B2_TRY(enqueue_iteration(c, m, false));
    B2_TRY(read_energy(c, m, t, efix));
    mark_valid(c, LABELS);
    return B2TEX_OK;
}

// Iterations t_begin .. max_iterations (fine, or on the contracted MRF) without a host round trip per iteration: the host
// queues iterations ahead of the device; the stop rule is evaluated on the device and turns the launches that are already
// queued behind it into no-ops.  With peers attached (mrf_mg_export / mrf_mg_import) every rank runs this same loop; the
// ranks meet inside the kernels.
// t_last: the last iteration to queue, if before max_iterations.
enum class Phase { fine, coarse, spanning };
int run_phase(b2tex_ctx *c, uint32_t t_begin, uint32_t t_ref, Phase phase, uint32_t t_last = 0xFFFFFFFFu)
{
    cudaStream_t s = c->stream;
    const uint32_t max_it = std::min(c->mrf_params.max_iterations, t_last);
    constexpr int LAG = 3;   // iterations queued beyond the last one whose stop flag the host has seen
    cudaEvent_t ev[LAG + 1];
    for (auto &e : ev) B2_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    volatile uint32_t *hf = c->mrf_host_flags;
    int rc = B2TEX_OK;
    for (uint32_t t = t_begin; t <= max_it; ++t) {
        Mrf m = make_mrf(c, t);
        rc = phase == Phase::coarse ? enqueue_coarse_iteration(c, t, t_ref)
             : phase == Phase::spanning ? enqueue_spanning_iteration(c, m, t_ref) : enqueue_iteration(c, m, true, t_ref);
        if (rc != B2TEX_OK) break;
        const int slot = (int)(t % (LAG + 1));
        if (cudaMemcpyAsync((void *)&hf[slot], m.state + ST_STOP, 4, cudaMemcpyDeviceToHost, s) != cudaSuccess ||
            cudaEventRecord(ev[slot], s) != cudaSuccess) {
            set_error("view selection: %s", cudaGetErrorString(cudaGetLastError()));
            rc = B2TEX_ERR_CUDA;
            break;
        }
        if (t - t_begin >= (uint32_t)LAG) {
            const int w = (int)((t - LAG) % (LAG + 1));
            if (cudaEventSynchronize(ev[w]) != cudaSuccess) { set_error("view selection: %s", cudaGetErrorString(cudaGetLastError())); rc = B2TEX_ERR_CUDA; break; }
            if (hf[w]) break;   // the rule fired LAG iterations ago; what is queued behind it returns at once
        }
    }
    if (cudaStreamSynchronize(s) != cudaSuccess && rc == B2TEX_OK) {
        set_error("view selection: %s", cudaGetErrorString(cudaGetLastError()));
        rc = B2TEX_ERR_CUDA;
    }
    for (auto &e : ev) cudaEventDestroy(e);
    return rc;
}

// last iteration of the phase that started after t_ref
int phase_end(b2tex_ctx *c, uint32_t t_ref, uint32_t *t_end)
{
    uint32_t st[2];
    B2_CUDA(cudaMemcpyAsync(st, c->mrf_state.p + ST_STOP, sizeof(st), cudaMemcpyDeviceToHost, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    static_assert(ST_DONE == ST_STOP + 1, "state layout");
    *t_end = t_ref + (st[0] ? st[0] : st[1]);
    return B2TEX_OK;
}

// The multilevel schedule of oracle/mrf_multilevel.c, after the first fine phase (which started after *t_ref): contract
// the labeling, run the BCD on the contracted MRF from the current labels (every iteration projected, the trace and the
// stop rule on fine energies, window restarted), and go back to a fine phase while the coarse phase strictly lowered the
// energy.
int run_multilevel(b2tex_ctx *c, b2tex_mrf_info *info, uint32_t *t_ref)
{
    const uint32_t max_it = c->mrf_params.max_iterations;
    const Mrf m = make_mrf(c, 0);
    uint32_t t = 0;
    B2_TRY(phase_end(c, *t_ref, &t));
    while (t < max_it) {
        int64_t before = 0, after = 0;
        B2_TRY(read_energy(c, m, t, &before));
        uint32_t n = 0;
        {
            ScopedTimer tc(c, "mrf_ml.contract");
            B2_TRY(mrf_contract(c, &n));
            if (n) B2_LAUNCH k_build_adj4<<<(n + 255) / 256, 256, 0, c->stream>>>(n, c->ml_cadj_ptr.p, c->ml_cadj_idx.p, c->ml_cadj4.p);
            B2_KERNEL_CHECK();
        }
        info->coarse_nodes = n;
        B2_CUDA(cudaMemsetAsync(m.state + ST_STOP, 0, sizeof(uint32_t), c->stream));
        B2_TRY(run_phase(c, t + 1, t, Phase::coarse));
        *t_ref = t;
        uint32_t t2 = 0;
        B2_TRY(phase_end(c, t, &t2));
        B2_TRY(read_energy(c, m, t2, &after));
        if (!(after < before)) break;
        info->multilevel_passes++;
        if (t2 >= max_it) break;
        B2_CUDA(cudaMemsetAsync(m.state + ST_STOP, 0, sizeof(uint32_t), c->stream));
        B2_TRY(run_phase(c, t2 + 1, t2, Phase::fine));
        *t_ref = t2;
        B2_TRY(phase_end(c, t2, &t));
    }
    return B2TEX_OK;
}

// The spanning phase of oracle/mrf_mapmap.c: every n spanning iterations are queued without a host round trip, and one
// multilevel step follows them unless the stop rule has fired or the budget is spent.  Iteration numbers go on across both.
int run_spanning_with_steps(b2tex_ctx *c, uint32_t n, b2tex_mrf_info *info)
{
    const uint32_t max_it = c->mrf_params.max_iterations;
    for (uint32_t t = 1; t <= max_it;) {
        const uint32_t last = n - 1u >= max_it - t ? max_it : t + n - 1u;
        B2_TRY(run_phase(c, t, 0, Phase::spanning, last));   // ends with a stream synchronisation
        uint32_t stop = 0;
        B2_CUDA(cudaMemcpyAsync(&stop, c->mrf_state.p + ST_STOP, sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
        B2_CUDA(cudaStreamSynchronize(c->stream));
        if (stop || last >= max_it) break;
        uint32_t nodes = 0;
        B2_TRY(enqueue_multilevel_step(c, last + 1u, 0, &nodes));
        info->coarse_nodes = nodes;
        t = last + 2u;
    }
    return B2TEX_OK;
}

// The whole run: init, with use_spanning_tree the spanning phase, the iterations on induced forests (run_phase), and with
// use_multilevel the multilevel schedule (run_multilevel).
int mrf_run(b2tex_ctx *c, const b2tex_mrf_params *p, b2tex_mrf_info *info, double *trace)
{
    info->multilevel_passes = 0;
    info->coarse_nodes = 0;
    info->spanning_tree_iterations = 0;
    info->spanning_tree_rejected = 0;
    info->multilevel_steps = 0;
    info->multilevel_steps_rejected = 0;
    const uint32_t every = p->spanning_tree_multilevel_after_n_iterations;
    if (every && (!p->use_spanning_tree || !p->use_multilevel)) {
        set_error("view selection: spanning_tree_multilevel_after_n_iterations = %u needs use_spanning_tree = 1 and "
                  "use_multilevel = 1 (%u, %u)", every, p->use_spanning_tree, p->use_multilevel);
        return B2TEX_ERR_ARG;
    }
    if ((p->use_multilevel || p->use_spanning_tree) &&
        ((p->num_parts ? p->num_parts : 1) > 1 || mg_active(c) || c->face_begin != 0 || c->face_end != c->F)) {
        set_error("%s view selection: one GPU and the whole mesh only (num_parts %u, %s, face range %u..%u of %u)",
                  p->use_spanning_tree ? "spanning-tree" : "multilevel", p->num_parts,
                  mg_active(c) ? "peers attached" : "no peers", c->face_begin, c->face_end, c->F);
        return B2TEX_ERR_UNSUPPORTED;
    }
    int64_t e0 = 0;
    B2_TRY(mrf_init(c, p, &e0));
    info->tree_group = (uint32_t)c->mrf_group;
    info->tree_cap = c->mrf_tree_cap;
    info->label_mask_words = c->mrf_mask_words;
    info->global_trees = 0;
    cudaStream_t s = c->stream;
    const uint32_t max_it = p->max_iterations, window = p->window ? p->window : 1u;
    const bool mg = mg_active(c);
    info->sweep_bytes = 14ull * c->nnz + 20ull * c->F;
    if (c->face_end <= c->face_begin && !mg) {   // nothing owned: the energy is constant, the stop rule fires at `window`
        const uint32_t t_end = std::min(window, max_it);
        info->iterations = t_end; info->unseen = 0;
        info->energy_initial = info->energy_final = (double)e0 / 4294967296.0;
        if (trace) for (uint32_t t = 0; t <= t_end; ++t) trace[t] = info->energy_initial;
        return B2TEX_OK;
    }
    invalidate(c, LABELS);   // until the iterations below have finished without error
    uint32_t t_ref = 0;   // the stop rule's reference iteration of the last phase: ST_STOP / ST_DONE count from it
    if (p->use_spanning_tree) {
        if (every) B2_TRY(run_spanning_with_steps(c, every, info));
        else B2_TRY(run_phase(c, 1, 0, Phase::spanning));
        uint32_t t_sp = 0;
        B2_TRY(phase_end(c, 0, &t_sp));
        info->spanning_tree_iterations = t_sp;
        if (t_sp < max_it) {   // the acyclic phase from those labels, window restarted
            B2_CUDA(cudaMemsetAsync(c->mrf_state.p + ST_STOP, 0, sizeof(uint32_t), s));
            B2_TRY(run_phase(c, t_sp + 1, t_sp, Phase::fine));
            t_ref = t_sp;
        }
    } else {
        B2_TRY(run_phase(c, 1, 0, Phase::fine));
    }
    if (p->use_multilevel && !every) B2_TRY(run_multilevel(c, info, &t_ref));   // with steps, the acyclic phase is the last
    Mrf m = make_mrf(c, 0);
    if (mg) {   // one all-gather of the final labels by peer stores: seam leveling assembles its system on every rank
        MrfPeers pr = make_peers(c);
        ScopedTimer tg(c, "mrf.label_allgather", 4.0 * (double)(m.ne - m.nb) * (pr.nranks - 1));
        B2_LAUNCH k_range_push<<<std::max(1, c->num_sms * 2), 256, 0, s>>>(m, pr);
        B2_LAUNCH k_mg_sync<<<1, 32, 0, s>>>(m, pr, c->mrf_mg->epoch + 2u * MRF_SLOTS + 4u, 2, max_it, 1u, 0.0f, 0xFFFFFFFFu, c->mrf_mg->elocal.p);
        B2_KERNEL_CHECK();
        c->mrf_mg->epoch += 2u * MRF_SLOTS + 8u;   // the same step on every rank, however many launches were queued
    }
    B2_LAUNCH k_label_check<<<std::max(1, c->num_sms * 4), 256, 0, s>>>(m);
    B2_KERNEL_CHECK();
    uint32_t st[ST_WORDS];
    std::vector<unsigned long long> efix((size_t)max_it + 2, 0ull);
    {   // through the pinned read-back area
        unsigned long long *pin_e = reinterpret_cast<unsigned long long *>(c->mrf_host_flags + 64);
        uint32_t *pin_s = c->mrf_host_flags + 64 + 2 * MRF_SLOTS;
        B2_CUDA(cudaMemcpyAsync(pin_s, c->mrf_state.p, ST_WORDS * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        B2_CUDA(cudaMemcpyAsync(pin_e, c->mrf_energy.p, ((size_t)max_it + 1) * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
        B2_CUDA(cudaStreamSynchronize(s));
        memcpy(st, pin_s, sizeof(st));
        memcpy(efix.data(), pin_e, ((size_t)max_it + 1) * sizeof(unsigned long long));
    }
    if (st[ST_ERR]) { set_error("multi-GPU view selection: %u cross-GPU barrier timeouts (a peer did not arrive)", st[ST_ERR]); return B2TEX_ERR_CUDA; }
    const uint32_t t_end = t_ref + (st[ST_STOP] ? st[ST_STOP] : st[ST_DONE]);   // ST_STOP == 0 only for max_iterations == 0
    info->iterations = t_end;
    info->energy_initial = (double)(int64_t)efix[0] / 4294967296.0;
    info->energy_final = (double)(int64_t)efix[t_end] / 4294967296.0;
    info->unseen = st[ST_UNSEEN];
    info->spanning_tree_rejected = st[ST_REJECTED] - st[ST_STEP_REJ];
    info->multilevel_steps = st[ST_STEPS];
    info->multilevel_steps_rejected = st[ST_STEP_REJ];
    info->global_trees = st[ST_SLOW];
    if (trace) for (uint32_t t = 0; t <= t_end; ++t) trace[t] = (double)(int64_t)efix[t] / 4294967296.0;
    // roofline accounting of k_tree: SURVEY 8d's sweep formula restricted to the nodes the launches processed
    unsigned long long fn, fz;
    memcpy(&fn, st + ST_FNODES, 8); memcpy(&fz, st + ST_FNNZ, 8);
    c->mrf_forest_nodes = fn; c->mrf_forest_nnz = fz; c->mrf_slow_trees = st[ST_SLOW];
    if (c->profile && t_end) {
        const double per = (14.0 * (double)fz + 20.0 * (double)fn) / (double)t_end;
        for (auto &k : c->timers) if (!strcmp(k.name, "mrf.k_tree") && k.bytes == 0.0) k.bytes = per;
    }
    if (c->mrf_dbg.n) {
        unsigned long long d[16];
        B2_TRY(c->mrf_dbg.download(d, 16, s));
        B2_CUDA(cudaStreamSynchronize(s));
        fprintf(stderr, "k_forest phases over %u iterations [us]: round0 %.1f seed %.1f growth %.1f alloc %.1f scatter %.1f\n", t_end,
                d[1] / 1e3, d[2] / 1e3, d[3] / 1e3, d[4] / 1e3, d[5] / 1e3);
        fprintf(stderr, "k_tree: trees through global memory %u, forest nodes %llu in %llu labels\n", st[ST_SLOW], fn, fz);
    }
    if (st[ST_BAD]) { set_error("Incorrect labeling"); return B2TEX_ERR_LABELING; }
    mark_valid(c, LABELS);
    return B2TEX_OK;
}

// fixed-point energy of the owned nodes with the labels currently in the context (a host-driven sharded run calls
// this after its own label exchange, so that cut edges see the neighbours' NEW labels)
int mrf_energy_only(b2tex_ctx *c, int64_t *efix)
{
    B2_TRY(require(c, MRF, "mrf_energy"));
    Mrf m = make_mrf(c, 1);
    const uint32_t slot = MRF_SLOTS - 1;   // scratch slot
    B2_CUDA(cudaMemsetAsync(m.efix + slot, 0, sizeof(unsigned long long), c->stream));
    if (m.ne > m.nb) B2_LAUNCH k_energy<<<std::max(1, c->num_sms * 8), 256, 0, c->stream>>>(m, m.efix + slot);
    B2_KERNEL_CHECK();
    return read_energy(c, m, slot, efix);
}

int mrf_sample_only(b2tex_ctx *c, const b2tex_mrf_params *p, uint32_t t, uint32_t *level_host)
{
    if (!(c->valid & MRF)) { int64_t e; B2_TRY(mrf_init(c, p, &e)); }
    c->mrf_params = *p;
    Mrf m = make_mrf(c, t);
    B2_TRY(c->mrf_queue.zero(c->stream));  // the same (iteration, round) stamps may be replayed
    if (m.ne > m.nb) B2_TRY(launch_forest(c, m, 0));
    B2_TRY(c->mrf_level.download(level_host, c->F, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    return B2TEX_OK;
}

// ---- peer block management (one process per GPU; the 64-byte cudaIpc handles travel through the caller) ----
void mrf_mg_free(b2tex_ctx *c)
{
    MrfMgState *g = c->mrf_mg;
    if (!g) return;
    if (c->labels.borrowed) { c->labels.release(); invalidate(c, LABELS); }
    for (uint32_t k = 0; k < (uint32_t)MRF_MAX_RANKS; ++k)
        if (g->opened[k] && g->peer[k]) cudaIpcCloseMemHandle(g->peer[k]);
    if (g->block) cudaFree(g->block);
    delete g;
    c->mrf_mg = nullptr;
}

// needs the mesh (F); from here on c->labels lives inside the peer-visible block
int mrf_mg_export(b2tex_ctx *c, uint32_t rank, uint32_t nranks, void *handle64)
{
    if (!c->F) { set_error("mrf_mg_export: set the mesh first"); return B2TEX_ERR_ARG; }
    if (nranks < 1 || nranks > (uint32_t)MRF_MAX_RANKS || rank >= nranks) { set_error("mrf_mg_export: at most %d ranks", MRF_MAX_RANKS); return B2TEX_ERR_ARG; }
    mrf_mg_free(c);
    MrfMgState *g = new MrfMgState();
    c->mrf_mg = g;
    g->F = c->F; g->rank = rank; g->nranks = nranks;
    const size_t bytes = mrf_block_bytes(c->F);
    B2_CUDA(cudaMalloc(&g->block, bytes));
    B2_CUDA(cudaMemsetAsync(g->block, 0, bytes, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    g->peer[rank] = g->block;
    c->labels.borrow((uint32_t *)g->block, c->F);
    invalidate(c, LABELS);
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    cudaIpcMemHandle_t h;
    memset(&h, 0, sizeof(h));
    if (nranks > 1) B2_CUDA(cudaIpcGetMemHandle(&h, g->block));
    memcpy(handle64, &h, 64);
    return B2TEX_OK;
}

int mrf_mg_import(b2tex_ctx *c, uint32_t peer_rank, const void *handle64)
{
    MrfMgState *g = c->mrf_mg;
    if (!g || peer_rank >= g->nranks) { set_error("mrf_mg_import: export first"); return B2TEX_ERR_ARG; }
    if (peer_rank == g->rank) return B2TEX_OK;
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    B2_CUDA(cudaIpcOpenMemHandle(&g->peer[peer_rank], h, cudaIpcMemLazyEnablePeerAccess));
    g->opened[peer_rank] = true;
    return B2TEX_OK;
}

// Peers inside ONE process (two contexts, e.g. two devices driven by threads, or two contexts on one device in the
// tests): no IPC handle is needed, the raw device pointer of the peer's block is attached instead.
int mrf_mg_attach(b2tex_ctx *c, uint32_t peer_rank, void *peer_block)
{
    MrfMgState *g = c->mrf_mg;
    if (!g || peer_rank >= g->nranks || !peer_block) { set_error("mrf_mg_attach: export first"); return B2TEX_ERR_ARG; }
    if (peer_rank != g->rank) g->peer[peer_rank] = peer_block;
    return B2TEX_OK;
}
void *mrf_mg_block(b2tex_ctx *c) { return c->mrf_mg ? c->mrf_mg->block : nullptr; }

}  // namespace b2
