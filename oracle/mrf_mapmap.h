/* oracle/mrf_mapmap.h -- TEST INFRASTRUCTURE (see oracle.h).
 *
 * mapMAP's schedule as texrecon configures it (view_selection.cpp:103-115: use_spanning_tree, use_multilevel,
 * spanning_tree_multilevel_after_n_iterations = 5, use_acyclic + force_acyclic): a multilevel step after every n-th
 * iteration of the spanning phase, then the acyclic phase.  Built on oracle/mrf_spanning.c, oracle/mrf_multilevel.c and
 * oracle/mrf.c, which it links unchanged.  csrc/mrf.cu reproduces it bit for bit.
 */
#ifndef ORC_MRF_MAPMAP_H
#define ORC_MRF_MAPMAP_H

#include "oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The DP of one spanning-tree iteration (orc_mrf_sample_spanning's forest, oracle/mrf_spanning.c's rules) with Potts
 * weights per adjacency slot, without acceptance: a fixed neighbour adds (l != x_w ? w : 0), a child's message is
 * min(h_c(l), min h_c + w(c, parent)).  weight NULL = unit weights: then every operation is the one of
 * orc_mrf_spanning_iteration's DP.  labels: in = the labels at the start, out = after the DP.  level_out, parent_out may be
 * NULL. */
void orc_mrf_spanning_sweep_w(uint32_t num_nodes, const uint32_t *adj_ptr, const uint32_t *adj_idx, const float *weight,
                              const uint64_t *ptr, const uint16_t *view, const float *cost, const orc_mrf_params *params,
                              uint32_t iteration, uint32_t *labels, uint32_t *level_out, uint32_t *parent_out);

/* What one multilevel step did.  The arrays are optional outputs (NULL to skip), each with room for num_faces entries:
 * region = node of every face, clabels = the coarse labels at the start, level / parent = the coarse spanning forest,
 * swept = the coarse labels after the DP, projected = the face labels after the DP (before acceptance). */
typedef struct {
    uint32_t num_nodes;
    uint32_t rejected;
    int64_t energy_before;         /* fine 32.32 energy at the start */
    int64_t energy_swept;          /* of the projected DP result */
    int64_t energy_after;          /* after acceptance: energy_swept, or energy_before if rejected */
    int64_t coarse_energy_after;   /* orc_coarse_energy_fixed of the coarse labels after acceptance */
    uint32_t *region, *clabels, *level, *parent, *swept, *projected;
} orc_mm_step;

/* One multilevel step of iteration t on `labels` (in: at its start, out: after it): contract (orc_mrf_contract), one
 * spanning-tree iteration with weighted Potts terms on the contracted MRF (seed of iteration t), projection onto the faces,
 * and acceptance on the fine energy (rejected: the coarse labels from the start are projected back). */
int orc_mrf_mapmap_step(uint32_t num_faces, const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint64_t *face_ptr,
                        const uint16_t *view, const float *cost, const orc_mrf_params *params, uint32_t iteration,
                        uint32_t *labels, orc_mm_step *step);

typedef struct {
    uint32_t iterations;                  /* all phases, numbered on from one phase to the next */
    uint32_t spanning_tree_iterations;    /* the spanning phase, its multilevel steps included */
    uint32_t spanning_tree_rejected;      /* spanning iterations that were rejected */
    uint32_t acyclic_iterations;          /* the acyclic phase */
    uint32_t multilevel_passes;           /* n == 0 only: the post-acyclic multilevel schedule */
    uint32_t coarse_nodes;                /* nodes of the last contraction */
    uint32_t multilevel_steps;            /* n > 0: multilevel steps inside the spanning phase */
    uint32_t multilevel_steps_rejected;   /* of those, the ones that were rejected */
    uint32_t identity_failures;           /* steps after which coarse != fine energy (must stay 0) */
    uint32_t pad;
    double energy_initial;
    double energy_final;
    uint64_t unseen;
} orc_mm_info;

/* n == 0: exactly orc_view_selection_st(use_spanning_tree, use_multilevel).  n > 0 (both flags required, else returns 2):
 * arg-min start; the spanning phase, where a multilevel step (next iteration number, its seed) follows every spanning
 * iteration whose count inside the phase is a multiple of n, unless the stop rule fired or max_iterations is reached --
 * every iteration, steps included, enters the trace and the stop rule's window; then the acyclic phase, window
 * restarted, and nothing after it.  trace: max_iterations + 1 entries.  num_parts > 1 returns 1. */
int orc_view_selection_mapmap(uint32_t num_faces, const uint32_t *adj_ptr, const uint32_t *adj_idx,
                              const uint64_t *face_ptr, const uint16_t *view, const float *cost,
                              const orc_mrf_params *params, uint32_t use_spanning_tree, uint32_t use_multilevel,
                              uint32_t n, uint32_t *labels_out, double *trace, orc_mm_info *info);

#ifdef __cplusplus
}
#endif
#endif
