/* oracle/mrf_spanning.h -- TEST INFRASTRUCTURE (see oracle.h).
 *
 * The spanning-tree step of view selection (mapMAP's use_spanning_tree, view_selection.cpp:103-111), restated on top of
 * the forest block-coordinate descent of oracle/mrf.c and composed with the multilevel schedule of
 * oracle/mrf_multilevel.c.  csrc/mrf.cu reproduces it bit for bit.
 */
#ifndef ORC_MRF_SPANNING_H
#define ORC_MRF_SPANNING_H

#include "oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* growth rounds of one spanning forest at most: MAX_LEVELS - 2 of csrc/mrf.cu, the bound alloc_mrf puts on `rounds` */
#define ORC_SPAN_MAX_ROUNDS 1022u

/* The spanning forest of iteration t: the acyclic sampler's round-0 roots, then BFS growth.  level[v] = join round
 * (0xFFFFFFFF not reached, 0xFFFFFFFE unseen), parent[v] = the level - 1 neighbour with the largest priority
 * (0xFFFFFFFF for roots and nodes outside the forest).  Returns the deepest level. */
uint32_t orc_mrf_sample_spanning(uint32_t num_faces, const uint32_t *adj_ptr, const uint32_t *adj_idx,
                                 const uint64_t *face_ptr, const orc_mrf_params *params, uint32_t iteration,
                                 uint32_t *level_out, uint32_t *parent_out);

/* One spanning-tree iteration on `labels` (in: the labels at its start, out: after it): exact DP on the spanning forest
 * with every non-tree neighbour fixed at its label from the start of the iteration, then acceptance.  level_out,
 * parent_out, swept_out (the labels of the DP before acceptance) may be NULL.  Returns 1 if the iteration raised the
 * 32.32 energy and was rejected (labels restored), else 0. */
int orc_mrf_spanning_iteration(uint32_t num_faces, const uint32_t *adj_ptr, const uint32_t *adj_idx,
                               const uint64_t *face_ptr, const uint16_t *view, const float *cost,
                               const orc_mrf_params *params, uint32_t iteration, uint32_t *labels, uint32_t *level_out,
                               uint32_t *parent_out, uint32_t *swept_out);

typedef struct {
    uint32_t iterations;                 /* all phases, numbered on from one phase to the next */
    uint32_t spanning_tree_iterations;   /* the spanning phase */
    uint32_t spanning_tree_rejected;     /* its iterations that were rejected */
    uint32_t acyclic_iterations;         /* the first acyclic phase */
    uint32_t multilevel_passes;
    uint32_t coarse_nodes;
    double energy_initial;
    double energy_final;
    uint64_t unseen;
} orc_st_info;

/* arg-min start, the spanning phase (use_spanning_tree), the acyclic phase (window restarted), then the multilevel
 * schedule (use_multilevel).  With use_spanning_tree = 0 the labels and trace are those of orc_view_selection_ml.
 * trace: max_iterations + 1 entries, the fine energy after every iteration.  num_parts > 1 returns 1. */
int orc_view_selection_st(uint32_t num_faces, const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint64_t *face_ptr,
                          const uint16_t *view, const float *cost, const orc_mrf_params *params,
                          uint32_t use_spanning_tree, uint32_t use_multilevel, uint32_t *labels_out, double *trace,
                          orc_st_info *info);

#ifdef __cplusplus
}
#endif
#endif
