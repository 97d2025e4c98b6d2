/* oracle/mrf_mapmap.c -- TEST INFRASTRUCTURE (see oracle.h, mrf_mapmap.h).
 *
 * texrecon runs mapMAP with use_spanning_tree, use_multilevel and spanning_tree_multilevel_after_n_iterations = 5: a
 * multilevel step inside the spanning phase, once every n spanning iterations.  mapMAP's own step is not available; this
 * is the project's definition [UPSTREAM-RECALL], built from the pieces the other two schedules define:
 *
 *   step      contract the current labels (orc_mrf_contract, unchanged); ONE spanning-tree iteration on the contracted MRF:
 *             orc_mrf_sample_spanning's roots and BFS growth on the coarse nodes (unseen regions are never in the forest),
 *             and the exact min-sum DP with weighted Potts terms -- a fixed neighbour adds (l != x_w ? w : 0), a child's
 *             message is min(h_c(l), min h_c + w(c, parent)), every non-tree seen neighbour is fixed at its label from the
 *             start of the step; projection onto the faces; if the fine 32.32 energy rose, the coarse labels from the start
 *             are projected back (the projection of a contraction reproduces the labels it was made from) and the step
 *             counts as rejected.
 *   schedule  arg-min start; spanning phase (t = 1 ..): after every spanning iteration whose count inside the phase is a
 *             multiple of n, a step with the next iteration number (its seed), unless the stop rule fired or max_iterations
 *             is reached.  A step's energy enters the trace and the stop rule's window like any iteration, but it does not
 *             count towards the next multiple of n.  Then the acyclic phase of oracle/mrf.c, window restarted, and nothing
 *             after it: the interleaved steps replace the post-acyclic multilevel schedule, the acyclic phase stays the last
 *             one (force_acyclic).  It runs at least `window` iterations unless the budget runs out, which is what
 *             min_acyclic_iterations = 5 asks with window = 5.
 */
#include "mrf_mapmap.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "mrf_multilevel.h"
#include "mrf_spanning.h"

#define NO_NODE 0xFFFFFFFFu

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

void orc_mrf_spanning_sweep_w(uint32_t F, const uint32_t *adj_ptr, const uint32_t *adj_idx, const float *wgt,
                              const uint64_t *ptr, const uint16_t *view, const float *cost, const orc_mrf_params *pr,
                              uint32_t t, uint32_t *labels, uint32_t *level_out, uint32_t *parent_out)
{
    const size_t Fa = F ? F : 1, nnz = ptr[F] ? ptr[F] : 1;
    uint32_t *level = (uint32_t *)malloc(sizeof(uint32_t) * Fa), *parent = (uint32_t *)malloc(sizeof(uint32_t) * Fa);
    uint32_t *order = (uint32_t *)malloc(sizeof(uint32_t) * Fa), *amin = (uint32_t *)malloc(sizeof(uint32_t) * Fa);
    uint32_t *lvl_ptr = (uint32_t *)malloc(sizeof(uint32_t) * (ORC_SPAN_MAX_ROUNDS + 2));
    float *H = (float *)malloc(sizeof(float) * nnz), *hminp1 = (float *)malloc(sizeof(float) * Fa);
    const uint32_t L = orc_mrf_sample_spanning(F, adj_ptr, adj_idx, ptr, pr, t, level, parent);
    memset(lvl_ptr, 0, sizeof(uint32_t) * (L + 2));
    for (uint32_t v = 0; v < F; ++v) if (level[v] <= L) lvl_ptr[level[v] + 1]++;
    for (uint32_t r = 0; r <= L; ++r) lvl_ptr[r + 1] += lvl_ptr[r];
    memcpy(amin, lvl_ptr, sizeof(uint32_t) * (L + 1));   /* fill positions; amin is free until the bottom-up pass */
    for (uint32_t v = 0; v < F; ++v) if (level[v] <= L) order[amin[level[v]]++] = v;
    for (int64_t r = (int64_t)L; r >= 0; --r) {
        for (uint32_t oi = lvl_ptr[r]; oi < lvl_ptr[r + 1]; ++oi) {
            const uint32_t v = order[oi];
            float hmin = INFINITY, wpar = 1.0f;
            uint32_t hidx = 0;
            if (wgt)
                for (uint32_t a = adj_ptr[v]; a < adj_ptr[v + 1]; ++a)
                    if (adj_idx[a] == parent[v]) wpar = wgt[a];
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
                        h = h + (lab != labels[w] ? (wgt ? wgt[a] : 1.0f) : 0.0f);
                    }
                }
                H[k] = h;
                if (h < hmin) { hmin = h; hidx = (uint32_t)(k - ptr[v]); }
            }
            hminp1[v] = hmin + wpar;
            amin[v] = hidx;
        }
    }
    for (uint32_t r = 0; r <= L; ++r) {
        for (uint32_t oi = lvl_ptr[r]; oi < lvl_ptr[r + 1]; ++oi) {
            const uint32_t v = order[oi];
            uint32_t best = (uint32_t)view[ptr[v] + amin[v]] + 1u;
            if (parent[v] != NO_NODE) {
                const uint32_t xp = labels[parent[v]];   /* assigned one level earlier */
                const int64_t j = find_label(ptr, view, v, xp);
                if (j >= 0 && H[j] <= hminp1[v]) best = xp;
            }
            labels[v] = best;
        }
    }
    if (level_out) memcpy(level_out, level, sizeof(uint32_t) * F);
    if (parent_out) memcpy(parent_out, parent, sizeof(uint32_t) * F);
    free(level); free(parent); free(order); free(amin); free(lvl_ptr); free(H); free(hminp1);
}

int orc_mrf_mapmap_step(uint32_t F, const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint64_t *ptr,
                        const uint16_t *view, const float *cost, const orc_mrf_params *pr, uint32_t t, uint32_t *labels,
                        orc_mm_step *st)
{
    orc_coarse_mrf c;
    orc_mrf_contract(F, adj_ptr, adj_idx, ptr, view, cost, labels, &c);
    const uint32_t n = c.num_nodes;
    uint32_t *old = (uint32_t *)malloc(sizeof(uint32_t) * (n ? n : 1));
    memcpy(old, c.labels, sizeof(uint32_t) * n);
    st->num_nodes = n;
    st->energy_before = orc_mrf_energy_fixed(F, adj_ptr, adj_idx, ptr, view, cost, labels);
    if (st->region) memcpy(st->region, c.region, sizeof(uint32_t) * F);
    if (st->clabels) memcpy(st->clabels, c.labels, sizeof(uint32_t) * n);
    orc_mrf_spanning_sweep_w(n, c.adj_ptr, c.adj_idx, c.weight, c.ptr, c.view, c.cost, pr, t, c.labels, st->level,
                             st->parent);
    if (st->swept) memcpy(st->swept, c.labels, sizeof(uint32_t) * n);
    for (uint32_t f = 0; f < F; ++f) labels[f] = c.labels[c.region[f]];
    if (st->projected) memcpy(st->projected, labels, sizeof(uint32_t) * F);
    st->energy_swept = orc_mrf_energy_fixed(F, adj_ptr, adj_idx, ptr, view, cost, labels);
    st->rejected = st->energy_swept > st->energy_before;
    st->energy_after = st->energy_swept;
    if (st->rejected) {
        memcpy(c.labels, old, sizeof(uint32_t) * n);
        for (uint32_t f = 0; f < F; ++f) labels[f] = c.labels[c.region[f]];
        st->energy_after = st->energy_before;
    }
    st->coarse_energy_after = orc_coarse_energy_fixed(&c, F, c.region);
    free(old);
    orc_coarse_free(&c);
    return 0;
}

static int stop_rule(const int64_t *efix, const orc_mrf_params *pr, uint32_t t, uint32_t t_ref)
{
    if (t - t_ref < pr->window) return 0;
    const double e0 = (double)efix[t - pr->window], e1 = (double)efix[t];   /* view_selection.cpp:84 */
    return e0 <= 0.0 || (e0 - e1) / e0 < (double)pr->ratio;
}

int orc_view_selection_mapmap(uint32_t F, const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint64_t *ptr,
                              const uint16_t *view, const float *cost, const orc_mrf_params *pr,
                              uint32_t use_spanning_tree, uint32_t use_multilevel, uint32_t n, uint32_t *labels,
                              double *trace, orc_mm_info *info)
{
    memset(info, 0, sizeof(*info));
    if (n == 0) {
        orc_st_info si;
        const int rc = orc_view_selection_st(F, adj_ptr, adj_idx, ptr, view, cost, pr, use_spanning_tree, use_multilevel,
                                             labels, trace, &si);
        info->iterations = si.iterations;
        info->spanning_tree_iterations = si.spanning_tree_iterations;
        info->spanning_tree_rejected = si.spanning_tree_rejected;
        info->acyclic_iterations = si.acyclic_iterations;
        info->multilevel_passes = si.multilevel_passes;
        info->coarse_nodes = si.coarse_nodes;
        info->energy_initial = si.energy_initial;
        info->energy_final = si.energy_final;
        info->unseen = si.unseen;
        return rc;
    }
    if (!use_spanning_tree || !use_multilevel) return 2;
    if (pr->num_parts > 1) return 1;
    int64_t *efix = (int64_t *)malloc(sizeof(int64_t) * (pr->max_iterations + 1));
    for (uint32_t i = 0; i < F; ++i) {   /* arg-min of the unaries (first minimum); unseen -> 0 */
        if (ptr[i + 1] == ptr[i]) { labels[i] = 0; ++info->unseen; continue; }
        uint64_t best = ptr[i];
        for (uint64_t k = ptr[i] + 1; k < ptr[i + 1]; ++k) if (cost[k] < cost[best]) best = k;
        labels[i] = (uint32_t)view[best] + 1u;
    }
    efix[0] = orc_mrf_energy_fixed(F, adj_ptr, adj_idx, ptr, view, cost, labels);
    info->energy_initial = orc_mrf_energy(F, adj_ptr, adj_idx, ptr, view, cost, labels);
    uint32_t t = 0, k = 0;
    while (t < pr->max_iterations) {   /* the spanning phase with its multilevel steps */
        ++t; ++k;
        const int rej = orc_mrf_spanning_iteration(F, adj_ptr, adj_idx, ptr, view, cost, pr, t, labels, NULL, NULL, NULL);
        efix[t] = rej ? efix[t - 1] : orc_mrf_energy_fixed(F, adj_ptr, adj_idx, ptr, view, cost, labels);
        info->spanning_tree_rejected += (uint32_t)rej;
        if (stop_rule(efix, pr, t, 0)) break;
        if (k % n == 0 && t < pr->max_iterations) {
            ++t;
            orc_mm_step st;
            memset(&st, 0, sizeof(st));
            orc_mrf_mapmap_step(F, adj_ptr, adj_idx, ptr, view, cost, pr, t, labels, &st);
            efix[t] = st.energy_after;
            info->multilevel_steps++;
            info->multilevel_steps_rejected += st.rejected;
            info->coarse_nodes = st.num_nodes;
            if (st.coarse_energy_after != st.energy_after) info->identity_failures++;
            if (stop_rule(efix, pr, t, 0)) break;
        }
    }
    info->spanning_tree_iterations = t;
    const uint32_t t_sp = t;
    for (uint32_t u = t_sp + 1; u <= pr->max_iterations; ++u) {   /* the acyclic phase, window restarted */
        orc_mrf_sweep(F, adj_ptr, adj_idx, NULL, ptr, view, cost, pr, u, labels);
        efix[u] = orc_mrf_energy_fixed(F, adj_ptr, adj_idx, ptr, view, cost, labels);
        t = u;
        if (stop_rule(efix, pr, u, t_sp)) break;
    }
    info->acyclic_iterations = t - t_sp;
    info->iterations = t;
    info->energy_final = orc_mrf_energy(F, adj_ptr, adj_idx, ptr, view, cost, labels);
    if (trace) for (uint32_t i = 0; i <= t; ++i) trace[i] = (double)efix[i] / 4294967296.0;
    free(efix);
    return 0;
}
