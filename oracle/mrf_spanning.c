/* oracle/mrf_spanning.c -- TEST INFRASTRUCTURE (see oracle.h, mrf_spanning.h).
 *
 * The induced forests of oracle/mrf.c leave about a third of the nodes out of every block.  The spanning-tree step solves
 * a spanning forest of the seen faces instead.  mapMAP's own step is not available; this is the project's definition:
 *
 *   sampler   iteration t uses prio_t(v) = mix32(v ^ iter_seed(seed, t)) as oracle/mrf.c does.  Roots are the acyclic
 *             sampler's round-0 roots (root candidates that beat every adjacent candidate; root_div == 0: the seen node
 *             with the largest priority).  In round r >= 1 every undecided seen node with a neighbour at level r - 1
 *             joins at level r, and its parent is the level r - 1 neighbour with the largest priority (a bijection: the
 *             parent is unique).  Growth stops when a round adds nobody or after ORC_SPAN_MAX_ROUNDS rounds; nodes not
 *             reached keep their labels.
 *   DP        oracle/mrf.c's exact min-sum DP (fp32, additions and minima only, adjacency order), where a child is a
 *             neighbour w with parent(w) == v, the parent is parent(v), and every other seen neighbour -- non-tree edges
 *             inside the tree and edges to other trees alike -- is fixed at its label from the start of the iteration
 *             (mapMAP's tree DP treats such neighbours as dependencies the same way [UPSTREAM-RECALL]).
 *   accept    conditioning non-tree edges on old labels does not guarantee descent: if the 32.32 energy after the sweep
 *             is above the one before, the labels from the start of the iteration come back and the iteration counts
 *             as rejected.  The trace is non-increasing.
 *   schedule  arg-min start; spanning phase (t = 1 ..) until StopWhenReturnsDiminish fires or max_iterations; the
 *             acyclic phase of oracle/mrf.c from those labels, window restarted; then oracle/mrf_multilevel.c's
 *             multilevel schedule if use_multilevel.  Iteration numbers, seeds and the budget continue across phases.
 */
#include "mrf_spanning.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "mrf_multilevel.h"

#define LVL_NONE 0xFFFFFFFFu
#define LVL_DEAD 0xFFFFFFFEu
#define NO_NODE 0xFFFFFFFFu

static inline uint32_t mix32(uint32_t x)
{
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}
static inline uint32_t iter_seed(uint32_t seed, uint32_t t) { return mix32(seed + 0x9E3779B9u * (t + 1u)); }
static inline uint32_t prio(uint32_t v, uint32_t seed_t) { return mix32(v ^ seed_t); }
static inline int root_cand(uint32_t v, uint32_t seed_t, uint32_t root_div)
{
    return mix32(prio(v, seed_t) ^ 0x68E31DA4u) % root_div == 0;
}
static inline uint32_t root_div_eff(uint32_t root_div, uint32_t F)
{
    if (root_div == 0) return 0;
    uint32_t cap = F / 8u; if (cap < 1u) cap = 1u;
    return root_div < cap ? root_div : cap;
}
static inline int seen(const uint64_t *ptr, uint32_t v) { return ptr[v + 1] > ptr[v]; }

static inline int64_t find_label(const uint64_t *ptr, const uint16_t *view, uint32_t w, uint32_t lab)
{
    uint64_t lo = ptr[w], hi = ptr[w + 1];
    while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        uint32_t l = (uint32_t)view[mid] + 1u;
        if (l < lab) lo = mid + 1; else hi = mid;
    }
    if (lo < ptr[w + 1] && (uint32_t)view[lo] + 1u == lab) return (int64_t)lo;
    return -1;
}

uint32_t orc_mrf_sample_spanning(uint32_t F, const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint64_t *ptr,
                                 const orc_mrf_params *pr, uint32_t t, uint32_t *level, uint32_t *parent)
{
    const uint32_t seed_t = iter_seed(pr->seed, t), rdiv = root_div_eff(pr->root_div, F);
    uint32_t best_prio = 0;
    int have_best = 0;
    if (rdiv == 0)
        for (uint32_t v = 0; v < F; ++v)
            if (seen(ptr, v) && (!have_best || prio(v, seed_t) > best_prio)) { best_prio = prio(v, seed_t); have_best = 1; }
    for (uint32_t v = 0; v < F; ++v) {   /* round 0: the acyclic sampler's roots (one partition) */
        parent[v] = NO_NODE;
        if (!seen(ptr, v)) { level[v] = LVL_DEAD; continue; }
        const uint32_t pv = prio(v, seed_t);
        int is_root = rdiv ? root_cand(v, seed_t, rdiv) : (pv == best_prio);
        for (uint32_t a = adj_ptr[v]; a < adj_ptr[v + 1] && rdiv && is_root; ++a) {
            const uint32_t w = adj_idx[a];
            if (seen(ptr, w) && root_cand(w, seed_t, rdiv) && prio(w, seed_t) > pv) is_root = 0;
        }
        level[v] = is_root ? 0u : LVL_NONE;
    }
    uint32_t maxl = 0;
    for (uint32_t r = 1; r <= ORC_SPAN_MAX_ROUNDS; ++r) {
        int joined = 0;
        for (uint32_t v = 0; v < F; ++v) {
            if (level[v] != LVL_NONE) continue;
            uint32_t par = NO_NODE, pp = 0;
            for (uint32_t a = adj_ptr[v]; a < adj_ptr[v + 1]; ++a) {
                const uint32_t w = adj_idx[a];
                if (level[w] == r - 1u && (par == NO_NODE || prio(w, seed_t) > pp)) { par = w; pp = prio(w, seed_t); }
            }
            if (par != NO_NODE) { level[v] = r; parent[v] = par; joined = 1; }
        }
        if (!joined) break;
        maxl = r;
    }
    return maxl;
}

typedef struct {
    float *H, *hminp1;
    uint32_t *amin, *level, *parent, *order, *lvl_ptr, *old;
} scratch_t;

static void scratch_alloc(scratch_t *s, uint32_t F, uint64_t nnz)
{
    s->H = (float *)malloc(sizeof(float) * (nnz ? nnz : 1));
    s->hminp1 = (float *)malloc(sizeof(float) * (F ? F : 1));
    s->amin = (uint32_t *)malloc(sizeof(uint32_t) * (F ? F : 1));
    s->level = (uint32_t *)malloc(sizeof(uint32_t) * (F ? F : 1));
    s->parent = (uint32_t *)malloc(sizeof(uint32_t) * (F ? F : 1));
    s->order = (uint32_t *)malloc(sizeof(uint32_t) * (F ? F : 1));
    s->lvl_ptr = (uint32_t *)malloc(sizeof(uint32_t) * (ORC_SPAN_MAX_ROUNDS + 2));
    s->old = (uint32_t *)malloc(sizeof(uint32_t) * (F ? F : 1));
}
static void scratch_free(scratch_t *s)
{
    free(s->H); free(s->hminp1); free(s->amin); free(s->level); free(s->parent); free(s->order); free(s->lvl_ptr);
    free(s->old);
}

/* the DP on the spanning forest of iteration t; s->old receives the labels at the start */
static void sweep(uint32_t F, const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint64_t *ptr, const uint16_t *view,
                  const float *cost, const orc_mrf_params *pr, uint32_t t, uint32_t *labels, scratch_t *s)
{
    uint32_t *level = s->level, *parent = s->parent, *order = s->order, *lvl_ptr = s->lvl_ptr;
    float *H = s->H, *hminp1 = s->hminp1;
    const uint32_t L = orc_mrf_sample_spanning(F, adj_ptr, adj_idx, ptr, pr, t, level, parent);
    memcpy(s->old, labels, sizeof(uint32_t) * F);
    memset(lvl_ptr, 0, sizeof(uint32_t) * (L + 2));
    for (uint32_t v = 0; v < F; ++v) if (level[v] <= L) lvl_ptr[level[v] + 1]++;
    for (uint32_t r = 0; r <= L; ++r) lvl_ptr[r + 1] += lvl_ptr[r];
    {
        uint32_t *pos = s->amin;   /* free until the bottom-up pass */
        memcpy(pos, lvl_ptr, sizeof(uint32_t) * (L + 1));
        for (uint32_t v = 0; v < F; ++v) if (level[v] <= L) order[pos[level[v]]++] = v;
    }
    for (int64_t r = (int64_t)L; r >= 0; --r) {
        for (uint32_t oi = lvl_ptr[r]; oi < lvl_ptr[r + 1]; ++oi) {
            const uint32_t v = order[oi];
            float hmin = INFINITY;
            uint32_t hidx = 0;
            for (uint64_t k = ptr[v]; k < ptr[v + 1]; ++k) {
                const uint32_t lab = (uint32_t)view[k] + 1u;
                float h = cost[k];
                for (uint32_t a = adj_ptr[v]; a < adj_ptr[v + 1]; ++a) {
                    const uint32_t w = adj_idx[a];
                    if (!seen(ptr, w)) continue;
                    if (parent[w] == v) {   /* child */
                        float msg = hminp1[w];
                        const int64_t j = find_label(ptr, view, w, lab);
                        if (j >= 0 && H[j] < msg) msg = H[j];
                        h = h + msg;
                    } else if (w != parent[v]) {   /* fixed: every label is still the one from the start */
                        h = h + (lab != labels[w] ? 1.0f : 0.0f);
                    }
                }
                H[k] = h;
                if (h < hmin) { hmin = h; hidx = (uint32_t)(k - ptr[v]); }
            }
            hminp1[v] = hmin + 1.0f;
            s->amin[v] = hidx;
        }
    }
    for (uint32_t r = 0; r <= L; ++r) {
        for (uint32_t oi = lvl_ptr[r]; oi < lvl_ptr[r + 1]; ++oi) {
            const uint32_t v = order[oi];
            uint32_t best = (uint32_t)view[ptr[v] + s->amin[v]] + 1u;
            if (parent[v] != NO_NODE) {
                const uint32_t xp = labels[parent[v]];   /* assigned one level earlier */
                const int64_t j = find_label(ptr, view, v, xp);
                if (j >= 0 && H[j] <= hminp1[v]) best = xp;
            }
            labels[v] = best;
        }
    }
}

/* sweep + acceptance against e_prev; returns the energy after the iteration, *rejected = 1 if the labels came back */
static int64_t iterate(uint32_t F, const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint64_t *ptr,
                       const uint16_t *view, const float *cost, const orc_mrf_params *pr, uint32_t t, uint32_t *labels,
                       int64_t e_prev, scratch_t *s, int *rejected)
{
    sweep(F, adj_ptr, adj_idx, ptr, view, cost, pr, t, labels, s);
    const int64_t e = orc_mrf_energy_fixed(F, adj_ptr, adj_idx, ptr, view, cost, labels);
    *rejected = e > e_prev;
    if (!*rejected) return e;
    memcpy(labels, s->old, sizeof(uint32_t) * F);
    return e_prev;
}

int orc_mrf_spanning_iteration(uint32_t F, const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint64_t *ptr,
                               const uint16_t *view, const float *cost, const orc_mrf_params *pr, uint32_t t,
                               uint32_t *labels, uint32_t *level_out, uint32_t *parent_out, uint32_t *swept_out)
{
    scratch_t s;
    scratch_alloc(&s, F, ptr[F]);
    const int64_t e_prev = orc_mrf_energy_fixed(F, adj_ptr, adj_idx, ptr, view, cost, labels);
    sweep(F, adj_ptr, adj_idx, ptr, view, cost, pr, t, labels, &s);
    if (swept_out) memcpy(swept_out, labels, sizeof(uint32_t) * F);
    const int rejected = orc_mrf_energy_fixed(F, adj_ptr, adj_idx, ptr, view, cost, labels) > e_prev;
    if (rejected) memcpy(labels, s.old, sizeof(uint32_t) * F);
    if (level_out) memcpy(level_out, s.level, sizeof(uint32_t) * F);
    if (parent_out) memcpy(parent_out, s.parent, sizeof(uint32_t) * F);
    scratch_free(&s);
    return rejected;
}

/* ---- the schedule ---- */
typedef struct {
    uint32_t F;
    const uint32_t *adj_ptr, *adj_idx;
    const uint64_t *ptr;
    const uint16_t *view;
    const float *cost;
    const orc_mrf_params *pr;
    uint32_t *labels;
    int64_t *efix;
    scratch_t *s;
    uint32_t rejected;
} run_t;

static int stop_rule(const run_t *run, uint32_t t, uint32_t t_ref)
{
    if (t - t_ref < run->pr->window) return 0;
    const double e0 = (double)run->efix[t - run->pr->window], e1 = (double)run->efix[t];   /* view_selection.cpp:84 */
    return e0 <= 0.0 || (e0 - e1) / e0 < (double)run->pr->ratio;
}

/* iterations t_begin.. of one phase (stop rule window restarted at t_ref): spanning (kind 0), acyclic on the faces
 * (kind 1), or acyclic on the contracted MRF c, projected onto the faces (kind 2).  Returns the last iteration run. */
static uint32_t run_phase(run_t *run, int kind, const orc_coarse_mrf *c, uint32_t t_begin, uint32_t t_ref)
{
    const orc_mrf_params *pr = run->pr;
    uint32_t last = t_begin - 1;
    for (uint32_t t = t_begin; t <= pr->max_iterations; ++t) {
        if (kind == 0) {
            int rej = 0;
            run->efix[t] = iterate(run->F, run->adj_ptr, run->adj_idx, run->ptr, run->view, run->cost, pr, t, run->labels,
                                   run->efix[t - 1], run->s, &rej);
            run->rejected += (uint32_t)rej;
        } else {
            if (kind == 1) {
                orc_mrf_sweep(run->F, run->adj_ptr, run->adj_idx, NULL, run->ptr, run->view, run->cost, pr, t, run->labels);
            } else {
                orc_mrf_sweep(c->num_nodes, c->adj_ptr, c->adj_idx, c->weight, c->ptr, c->view, c->cost, pr, t, c->labels);
                for (uint32_t f = 0; f < run->F; ++f) run->labels[f] = c->labels[c->region[f]];
            }
            run->efix[t] = orc_mrf_energy_fixed(run->F, run->adj_ptr, run->adj_idx, run->ptr, run->view, run->cost,
                                                run->labels);
        }
        last = t;
        if (stop_rule(run, t, t_ref)) break;
    }
    return last;
}

int orc_view_selection_st(uint32_t F, const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint64_t *ptr,
                          const uint16_t *view, const float *cost, const orc_mrf_params *pr, uint32_t use_spanning_tree,
                          uint32_t use_multilevel, uint32_t *labels, double *trace, orc_st_info *info)
{
    memset(info, 0, sizeof(*info));
    if (pr->num_parts > 1) return 1;
    scratch_t s;
    scratch_alloc(&s, F, ptr[F]);
    int64_t *efix = (int64_t *)malloc(sizeof(int64_t) * (pr->max_iterations + 1));
    for (uint32_t i = 0; i < F; ++i) {   /* arg-min of the unaries (first minimum); unseen -> 0 */
        if (ptr[i + 1] == ptr[i]) { labels[i] = 0; ++info->unseen; continue; }
        uint64_t best = ptr[i];
        for (uint64_t k = ptr[i] + 1; k < ptr[i + 1]; ++k) if (cost[k] < cost[best]) best = k;
        labels[i] = (uint32_t)view[best] + 1u;
    }
    efix[0] = orc_mrf_energy_fixed(F, adj_ptr, adj_idx, ptr, view, cost, labels);
    info->energy_initial = orc_mrf_energy(F, adj_ptr, adj_idx, ptr, view, cost, labels);
    run_t run = {F, adj_ptr, adj_idx, ptr, view, cost, pr, labels, efix, &s, 0};
    uint32_t t = 0;
    if (use_spanning_tree) {
        t = run_phase(&run, 0, NULL, 1, 0);
        info->spanning_tree_iterations = t;
        info->spanning_tree_rejected = run.rejected;
    }
    const uint32_t t_sp = t;
    t = run_phase(&run, 1, NULL, t + 1, t);
    info->acyclic_iterations = t - t_sp;
    while (use_multilevel && t < pr->max_iterations) {   /* oracle/mrf_multilevel.c's loop */
        const int64_t before = efix[t];
        orc_coarse_mrf c;
        orc_mrf_contract(F, adj_ptr, adj_idx, ptr, view, cost, labels, &c);
        info->coarse_nodes = c.num_nodes;
        const uint32_t t2 = run_phase(&run, 2, &c, t + 1, t);
        orc_coarse_free(&c);
        if (!(efix[t2] < before)) { t = t2; break; }
        info->multilevel_passes++;
        t = run_phase(&run, 1, NULL, t2 + 1, t2);
    }
    info->iterations = t;
    info->energy_final = orc_mrf_energy(F, adj_ptr, adj_idx, ptr, view, cost, labels);
    if (trace) for (uint32_t i = 0; i <= t; ++i) trace[i] = (double)efix[i] / 4294967296.0;
    scratch_free(&s);
    free(efix);
    return 0;
}
