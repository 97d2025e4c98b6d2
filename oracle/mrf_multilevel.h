/* oracle/mrf_multilevel.h -- TEST INFRASTRUCTURE (see oracle.h).
 *
 * The multilevel schedule of view selection (mapMAP's use_multilevel, view_selection.cpp:103-115), restated on top of the
 * forest block-coordinate descent of oracle/mrf.c.  csrc/mrf.cu + csrc/mrf_multilevel.cu reproduce it bit for bit.
 */
#ifndef ORC_MRF_MULTILEVEL_H
#define ORC_MRF_MULTILEVEL_H

#include "oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The MRF contracted from a labeling: one node per connected component of the face graph restricted to edges whose
 * faces carry the same label, numbered in the order of the component's lowest face id. */
typedef struct {
    uint32_t num_nodes;
    uint32_t *region;        /* [F] node of every face */
    uint32_t *size;          /* [n] faces per node */
    uint32_t *labels;        /* [n] the label of the node's faces */
    uint64_t *ptr;           /* [n + 1] label lists: the intersection of the members' lists (empty for unseen regions) */
    uint16_t *view;          /* [ptr[n]] ascending */
    float *cost;             /* [ptr[n]] sum of the members' costs, fp32, in ascending face order from 0.0f */
    int64_t *cost_fixed;     /* [ptr[n]] sum of the members' 32.32 fixed-point costs */
    uint32_t *adj_ptr;       /* [n + 1] symmetric CSR, neighbours ascending */
    uint32_t *adj_idx;
    float *weight;           /* [adj_ptr[n]] number of fine adjacency entries between the two nodes (from one side) */
} orc_coarse_mrf;

int orc_mrf_contract(uint32_t num_faces, const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint64_t *face_ptr,
                     const uint16_t *view, const float *cost, const uint32_t *labels, orc_coarse_mrf *out);
void orc_coarse_free(orc_coarse_mrf *c);
/* 32.32 energy of the coarse labeling c->labels: unaries of the seen nodes + weight of every cut edge between seen
 * nodes + one per unseen FACE (the constant of the fixed regions).  Equals orc_mrf_energy_fixed of the projection. */
int64_t orc_coarse_energy_fixed(const orc_coarse_mrf *c, uint32_t num_faces, const uint32_t *face_region);

/* one iteration of the forest BCD (single partition) with Potts weights per adjacency slot (NULL = unit weights) */
int orc_mrf_sweep(uint32_t num_nodes, const uint32_t *adj_ptr, const uint32_t *adj_idx, const float *weight,
                  const uint64_t *ptr, const uint16_t *view, const float *cost, const orc_mrf_params *params,
                  uint32_t iteration, uint32_t *labels);

typedef struct {
    uint32_t iterations;            /* fine and coarse, numbered on from one phase to the next */
    uint32_t first_phase_iterations;
    uint32_t multilevel_passes;     /* contractions whose coarse solve lowered the energy */
    uint32_t coarse_nodes;          /* nodes of the last contraction */
    uint32_t contractions;
    uint32_t identity_failures;     /* contractions after which fine != coarse + constant energy (must stay 0) */
    double energy_initial;
    double energy_final;
    uint64_t unseen;
} orc_ml_info;

/* use_multilevel = 0 runs exactly orc_view_selection.  labels_first_phase (or NULL) receives the labels at the end of the
 * first fine phase.  trace: max_iterations + 1 entries, the fine energy after every iteration. */
int orc_view_selection_ml(uint32_t num_faces, const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint64_t *face_ptr,
                          const uint16_t *view, const float *cost, const orc_mrf_params *params, uint32_t use_multilevel,
                          uint32_t *labels_out, uint32_t *labels_first_phase, double *trace, orc_ml_info *info);

#ifdef __cplusplus
}
#endif
#endif
