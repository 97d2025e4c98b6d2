/* oracle/mrf_multilevel.c -- TEST INFRASTRUCTURE (see oracle.h, mrf_multilevel.h).
 *
 * Node-wise descent under a Potts term cannot relabel a whole same-label region at once: every face of the region pays
 * the boundary cost alone.  The multilevel step contracts every such region into one node and runs the same forest
 * block-coordinate descent (oracle/mrf.c) on the smaller graph, with Potts weights = the number of fine edges between
 * two regions.  mapMAP's own schedule is not available; this is the project's definition:
 *
 *   1. fine phase: oracle/mrf.c's loop until StopWhenReturnsDiminish fires (window restarted at the phase's start) or
 *      max_iterations is reached.  The first fine phase is exactly orc_view_selection.
 *   2. contract the labeling (orc_mrf_contract).  Unseen regions (empty lists, label 0) stay fixed.
 *   3. coarse phase: the same BCD on the coarse MRF with weighted Potts terms, from the current labels; iteration numbers
 *      (hence seeds) and the max_iterations budget continue from the fine phase.  After every coarse iteration the
 *      labels are projected (labels[f] = coarse label of f's region) and the trace gets the FINE 32.32 energy, on which
 *      the stop rule runs, window restarted.
 *   4. if the energy at the end of the coarse phase is strictly lower than before step 2, go to 1; otherwise stop.
 *
 * The weighted DP is oracle/mrf.c's with `1.0f` replaced by the weight of the adjacency slot: a fixed neighbour adds
 * (l != x_w ? w : 0), a child's message is min(h_c(l), min h_c + w_parent).  With unit weights every operation is the
 * one of oracle/mrf.c.
 */
#include "mrf_multilevel.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#define FIX_ONE ((int64_t)1 << 32)

typedef struct {
    uint32_t F;
    const uint32_t *adj_ptr, *adj_idx;
    const float *wgt;              /* per adjacency slot, NULL = unit weights */
    const uint64_t *ptr;
    const uint16_t *view;
    const float *cost;
} graph_t;

static inline int seen(const graph_t *g, uint32_t v) { return g->ptr[v + 1] > g->ptr[v]; }
static inline float weight(const graph_t *g, uint32_t a) { return g->wgt ? g->wgt[a] : 1.0f; }

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

typedef struct {
    float *H, *hminp1;
    uint32_t *amin, *level, *order, *lvl_ptr, *pos;
} scratch_t;

/* one iteration of oracle/mrf.c's solver (single partition) on g, weighted */
static void sweep(const graph_t *g, const orc_mrf_params *pr, uint32_t t, uint32_t *labels, scratch_t *s)
{
    const uint32_t F = g->F, R = pr->rounds;
    uint32_t *level = s->level, *order = s->order, *lvl_ptr = s->lvl_ptr;
    float *H = s->H, *hminp1 = s->hminp1;
    orc_mrf_sample_forest(F, g->adj_ptr, g->adj_idx, g->ptr, pr, t, level);
    memset(lvl_ptr, 0, sizeof(uint32_t) * (R + 2));
    for (uint32_t v = 0; v < F; ++v) if (level[v] <= R) lvl_ptr[level[v] + 1]++;
    for (uint32_t r = 0; r <= R; ++r) lvl_ptr[r + 1] += lvl_ptr[r];
    memcpy(s->pos, lvl_ptr, sizeof(uint32_t) * (R + 2));
    for (uint32_t v = 0; v < F; ++v) if (level[v] <= R) order[s->pos[level[v]]++] = v;
    for (int64_t r = (int64_t)R; r >= 0; --r) {
        for (uint32_t oi = lvl_ptr[r]; oi < lvl_ptr[r + 1]; ++oi) {
            const uint32_t v = order[oi];
            float hmin = INFINITY, wpar = 1.0f;
            uint32_t hidx = 0;
            for (uint32_t a = g->adj_ptr[v]; a < g->adj_ptr[v + 1]; ++a) {
                const uint32_t w = g->adj_idx[a];
                if (seen(g, w) && level[w] < (uint32_t)r) wpar = weight(g, a);   /* the parent */
            }
            for (uint64_t k = g->ptr[v]; k < g->ptr[v + 1]; ++k) {
                const uint32_t lab = (uint32_t)g->view[k] + 1u;
                float h = g->cost[k];
                for (uint32_t a = g->adj_ptr[v]; a < g->adj_ptr[v + 1]; ++a) {
                    const uint32_t w = g->adj_idx[a];
                    if (!seen(g, w)) continue;
                    const uint32_t lw = level[w];
                    if (lw <= R) {
                        if (lw > (uint32_t)r) {   /* child */
                            float msg = hminp1[w];
                            const int64_t j = find_label(g->ptr, g->view, w, lab);
                            if (j >= 0 && H[j] < msg) msg = H[j];
                            h = h + msg;
                        }
                    } else {
                        h = h + (lab != labels[w] ? weight(g, a) : 0.0f);
                    }
                }
                H[k] = h;
                if (h < hmin) { hmin = h; hidx = (uint32_t)(k - g->ptr[v]); }
            }
            hminp1[v] = hmin + wpar;
            s->amin[v] = hidx;
        }
    }
    for (uint32_t r = 0; r <= R; ++r) {
        for (uint32_t oi = lvl_ptr[r]; oi < lvl_ptr[r + 1]; ++oi) {
            const uint32_t v = order[oi];
            uint32_t best = (uint32_t)g->view[g->ptr[v] + s->amin[v]] + 1u;
            if (r > 0) {
                for (uint32_t a = g->adj_ptr[v]; a < g->adj_ptr[v + 1]; ++a) {
                    const uint32_t w = g->adj_idx[a];
                    if (level[w] < r) {
                        const int64_t j = find_label(g->ptr, g->view, v, labels[w]);
                        if (j >= 0 && H[j] <= hminp1[v]) best = labels[w];
                        break;
                    }
                }
            }
            labels[v] = best;
        }
    }
}

int orc_mrf_sweep(uint32_t F, const uint32_t *adj_ptr, const uint32_t *adj_idx, const float *weight, const uint64_t *ptr,
                  const uint16_t *view, const float *cost, const orc_mrf_params *pr, uint32_t iteration, uint32_t *labels)
{
    const graph_t g = {F, adj_ptr, adj_idx, weight, ptr, view, cost};
    scratch_t s;
    const uint64_t nnz = ptr[F];
    s.H = (float *)malloc(sizeof(float) * (nnz ? nnz : 1));
    s.hminp1 = (float *)malloc(sizeof(float) * (F ? F : 1));
    s.amin = (uint32_t *)malloc(sizeof(uint32_t) * (F ? F : 1));
    s.level = (uint32_t *)malloc(sizeof(uint32_t) * (F ? F : 1));
    s.order = (uint32_t *)malloc(sizeof(uint32_t) * (F ? F : 1));
    s.lvl_ptr = (uint32_t *)malloc(sizeof(uint32_t) * (pr->rounds + 2));
    s.pos = (uint32_t *)malloc(sizeof(uint32_t) * (pr->rounds + 2));
    sweep(&g, pr, iteration, labels, &s);
    free(s.H); free(s.hminp1); free(s.amin); free(s.level); free(s.order); free(s.lvl_ptr); free(s.pos);
    return 0;
}

/* ---- contraction ---- */
int orc_mrf_contract(uint32_t F, const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint64_t *ptr,
                     const uint16_t *view, const float *cost, const uint32_t *labels, orc_coarse_mrf *c)
{
    memset(c, 0, sizeof(*c));
    uint32_t *region = (uint32_t *)malloc(sizeof(uint32_t) * (F ? F : 1));
    uint32_t *stack = (uint32_t *)malloc(sizeof(uint32_t) * (F ? F : 1));
    uint32_t n = 0;
    for (uint32_t v = 0; v < F; ++v) region[v] = UINT32_MAX;
    for (uint32_t s = 0; s < F; ++s) {   /* ascending start faces: nodes are numbered by their lowest face */
        if (region[s] != UINT32_MAX) continue;
        uint32_t top = 0;
        region[s] = n; stack[top++] = s;
        while (top) {
            const uint32_t v = stack[--top];
            for (uint32_t a = adj_ptr[v]; a < adj_ptr[v + 1]; ++a) {
                const uint32_t w = adj_idx[a];
                if (region[w] == UINT32_MAX && labels[w] == labels[v]) { region[w] = n; stack[top++] = w; }
            }
        }
        ++n;
    }
    /* members of every node, ascending */
    uint32_t *mptr = (uint32_t *)calloc((size_t)n + 1, sizeof(uint32_t));
    uint32_t *mem = stack;
    for (uint32_t v = 0; v < F; ++v) mptr[region[v] + 1]++;
    for (uint32_t r = 0; r < n; ++r) mptr[r + 1] += mptr[r];
    {
        uint32_t *fill = (uint32_t *)malloc(sizeof(uint32_t) * ((size_t)n + 1));
        memcpy(fill, mptr, sizeof(uint32_t) * ((size_t)n + 1));
        for (uint32_t v = 0; v < F; ++v) mem[fill[region[v]]++] = v;
        free(fill);
    }
    c->num_nodes = n;
    c->region = region;
    c->size = (uint32_t *)malloc(sizeof(uint32_t) * (n ? n : 1));
    c->labels = (uint32_t *)malloc(sizeof(uint32_t) * (n ? n : 1));
    c->ptr = (uint64_t *)calloc((size_t)n + 1, sizeof(uint64_t));
    const uint64_t nnz = ptr[F];
    c->view = (uint16_t *)malloc(sizeof(uint16_t) * (nnz ? nnz : 1));
    c->cost = (float *)malloc(sizeof(float) * (nnz ? nnz : 1));
    c->cost_fixed = (int64_t *)malloc(sizeof(int64_t) * (nnz ? nnz : 1));
    uint64_t e = 0;
    for (uint32_t r = 0; r < n; ++r) {
        const uint32_t root = mem[mptr[r]];
        c->size[r] = mptr[r + 1] - mptr[r];
        c->labels[r] = labels[root];
        for (uint64_t k = ptr[root]; k < ptr[root + 1]; ++k) {   /* the intersection of the lists */
            const uint32_t lab = (uint32_t)view[k] + 1u;
            float sum = 0.0f;
            int64_t fix = 0;
            int all = 1;
            for (uint32_t i = mptr[r]; i < mptr[r + 1] && all; ++i) {
                const int64_t j = find_label(ptr, view, mem[i], lab);
                if (j < 0) { all = 0; break; }
                sum = sum + cost[j];
                fix += (int64_t)((double)cost[j] * 4294967296.0);
            }
            if (!all) continue;
            c->view[e] = view[k]; c->cost[e] = sum; c->cost_fixed[e] = fix;
            ++e;
        }
        c->ptr[r + 1] = e;
    }
    /* edges: fine adjacency entries between different nodes, counted per (node, node) pair */
    uint32_t *cnt = (uint32_t *)calloc(n ? n : 1, sizeof(uint32_t));
    uint32_t *touched = (uint32_t *)malloc(sizeof(uint32_t) * (adj_ptr[F] ? adj_ptr[F] : 1));
    c->adj_ptr = (uint32_t *)calloc((size_t)n + 1, sizeof(uint32_t));
    c->adj_idx = (uint32_t *)malloc(sizeof(uint32_t) * (adj_ptr[F] ? adj_ptr[F] : 1));
    c->weight = (float *)malloc(sizeof(float) * (adj_ptr[F] ? adj_ptr[F] : 1));
    uint32_t ne = 0;
    for (uint32_t r = 0; r < n; ++r) {
        uint32_t nt = 0;
        for (uint32_t i = mptr[r]; i < mptr[r + 1]; ++i) {
            const uint32_t v = mem[i];
            for (uint32_t a = adj_ptr[v]; a < adj_ptr[v + 1]; ++a) {
                const uint32_t q = region[adj_idx[a]];
                if (q == r) continue;
                if (cnt[q]++ == 0) touched[nt++] = q;
            }
        }
        /* ascending neighbours: insertion sort (rows are short) */
        for (uint32_t i = 1; i < nt; ++i) {
            const uint32_t x = touched[i];
            uint32_t j = i;
            while (j > 0 && touched[j - 1] > x) { touched[j] = touched[j - 1]; --j; }
            touched[j] = x;
        }
        for (uint32_t i = 0; i < nt; ++i) {
            c->adj_idx[ne] = touched[i];
            c->weight[ne] = (float)cnt[touched[i]];
            cnt[touched[i]] = 0;
            ++ne;
        }
        c->adj_ptr[r + 1] = ne;
    }
    free(cnt); free(touched); free(mptr); free(mem);
    return 0;
}

void orc_coarse_free(orc_coarse_mrf *c)
{
    free(c->region); free(c->size); free(c->labels); free(c->ptr); free(c->view); free(c->cost); free(c->cost_fixed);
    free(c->adj_ptr); free(c->adj_idx); free(c->weight);
    memset(c, 0, sizeof(*c));
}

int64_t orc_coarse_energy_fixed(const orc_coarse_mrf *c, uint32_t F, const uint32_t *face_region)
{
    int64_t e = 0;
    for (uint32_t f = 0; f < F; ++f)
        if (c->ptr[face_region[f] + 1] == c->ptr[face_region[f]]) e += FIX_ONE;   /* unseen faces: one each */
    for (uint32_t r = 0; r < c->num_nodes; ++r) {
        if (c->ptr[r + 1] == c->ptr[r]) continue;
        const int64_t j = find_label(c->ptr, c->view, r, c->labels[r]);
        if (j < 0) return INT64_MIN;
        e += c->cost_fixed[j];
        for (uint32_t a = c->adj_ptr[r]; a < c->adj_ptr[r + 1]; ++a) {
            const uint32_t q = c->adj_idx[a];
            if (q > r && c->ptr[q + 1] > c->ptr[q] && c->labels[q] != c->labels[r]) e += (int64_t)c->weight[a] * FIX_ONE;
        }
    }
    return e;
}

/* ---- the schedule ---- */
typedef struct {
    const graph_t *fine;
    const orc_mrf_params *pr;
    uint32_t *labels;        /* fine labels */
    int64_t *efix;           /* [max_iterations + 1] */
    scratch_t *s;
} run_t;

/* iterations t_begin.. on g (the fine graph, or a coarse one whose labels `clabels` are projected through `region`
 * after every iteration); the stop rule compares efix[t - window] and efix[t] once t - t_ref >= window.
 * Returns the last iteration run (t_begin - 1 if none). */
static uint32_t run_phase(run_t *run, const graph_t *g, uint32_t *glabels, const uint32_t *region, uint32_t t_begin,
                          uint32_t t_ref)
{
    const orc_mrf_params *pr = run->pr;
    const graph_t *fg = run->fine;
    uint32_t last = t_begin - 1;
    for (uint32_t t = t_begin; t <= pr->max_iterations; ++t) {
        sweep(g, pr, t, glabels, run->s);
        if (region)
            for (uint32_t f = 0; f < fg->F; ++f) run->labels[f] = glabels[region[f]];
        run->efix[t] = orc_mrf_energy_fixed(fg->F, fg->adj_ptr, fg->adj_idx, fg->ptr, fg->view, fg->cost, run->labels);
        last = t;
        if (t - t_ref >= pr->window) {   /* StopWhenReturnsDiminish, view_selection.cpp:84 */
            const double e0 = (double)run->efix[t - pr->window], e1 = (double)run->efix[t];
            if (e0 <= 0.0 || (e0 - e1) / e0 < (double)pr->ratio) break;
        }
    }
    return last;
}

int orc_view_selection_ml(uint32_t F, const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint64_t *ptr,
                          const uint16_t *view, const float *cost, const orc_mrf_params *pr, uint32_t use_multilevel,
                          uint32_t *labels, uint32_t *labels_first, double *trace, orc_ml_info *info)
{
    memset(info, 0, sizeof(*info));
    if (pr->num_parts > 1) return 1;
    const graph_t fine = {F, adj_ptr, adj_idx, NULL, ptr, view, cost};
    const uint64_t nnz = ptr[F];
    scratch_t s;
    s.H = (float *)malloc(sizeof(float) * (nnz ? nnz : 1));
    s.hminp1 = (float *)malloc(sizeof(float) * (F ? F : 1));
    s.amin = (uint32_t *)malloc(sizeof(uint32_t) * (F ? F : 1));
    s.level = (uint32_t *)malloc(sizeof(uint32_t) * (F ? F : 1));
    s.order = (uint32_t *)malloc(sizeof(uint32_t) * (F ? F : 1));
    s.lvl_ptr = (uint32_t *)malloc(sizeof(uint32_t) * (pr->rounds + 2));
    s.pos = (uint32_t *)malloc(sizeof(uint32_t) * (pr->rounds + 2));
    int64_t *efix = (int64_t *)malloc(sizeof(int64_t) * (pr->max_iterations + 1));
    for (uint32_t i = 0; i < F; ++i) {   /* arg-min of the unaries (first minimum); unseen -> 0 */
        if (ptr[i + 1] == ptr[i]) { labels[i] = 0; ++info->unseen; continue; }
        uint64_t best = ptr[i];
        for (uint64_t k = ptr[i] + 1; k < ptr[i + 1]; ++k) if (cost[k] < cost[best]) best = k;
        labels[i] = (uint32_t)view[best] + 1u;
    }
    efix[0] = orc_mrf_energy_fixed(F, adj_ptr, adj_idx, ptr, view, cost, labels);
    info->energy_initial = orc_mrf_energy(F, adj_ptr, adj_idx, ptr, view, cost, labels);
    run_t run = {&fine, pr, labels, efix, &s};
    uint32_t t = run_phase(&run, &fine, labels, NULL, 1, 0);
    info->first_phase_iterations = t;
    if (labels_first) memcpy(labels_first, labels, sizeof(uint32_t) * F);
    while (use_multilevel && t < pr->max_iterations) {
        const int64_t before = efix[t];
        orc_coarse_mrf c;
        orc_mrf_contract(F, adj_ptr, adj_idx, ptr, view, cost, labels, &c);
        info->contractions++;
        info->coarse_nodes = c.num_nodes;
        const graph_t cg = {c.num_nodes, c.adj_ptr, c.adj_idx, c.weight, c.ptr, c.view, c.cost};
        const uint32_t t2 = run_phase(&run, &cg, c.labels, c.region, t + 1, t);
        if (orc_coarse_energy_fixed(&c, F, c.region) != efix[t2]) info->identity_failures++;
        orc_coarse_free(&c);
        if (!(efix[t2] < before)) { t = t2; break; }
        info->multilevel_passes++;
        t = run_phase(&run, &fine, labels, NULL, t2 + 1, t2);
    }
    info->iterations = t;
    info->energy_final = orc_mrf_energy(F, adj_ptr, adj_idx, ptr, view, cost, labels);
    if (trace) for (uint32_t i = 0; i <= t; ++i) trace[i] = (double)efix[i] / 4294967296.0;
    free(s.H); free(s.hminp1); free(s.amin); free(s.level); free(s.order); free(s.lvl_ptr); free(s.pos); free(efix);
    return 0;
}
