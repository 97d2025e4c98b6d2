/*
 * b2tex.h -- C ABI of the CUDA (sm_90a) mvs-texturing hot path (libb2tex.so).
 *
 * Drop-in boundary: the reference exposes this path as four C++ free functions in
 * libs/tex/texturing.h; each entry point below replaces one of them and is what a maintainer's
 * binding (see INTEGRATION.md, mvs-texturing_b200/tex/ for the C++ veneer that keeps the tex::
 * signatures) calls:
 *
 *   tex::calculate_data_costs   libs/tex/texturing.h:66-69  -> b2tex_calculate_data_costs
 *   tex::view_selection         libs/tex/texturing.h:79-80  -> b2tex_view_selection
 *   tex::global_seam_leveling   libs/tex/texturing.h:97-101 -> b2tex_global_seam_leveling
 *   (build_adjacency_graph      libs/tex/texturing.h:59-61  input of view_selection, passed as CSR)
 *   tex::prepare_mesh           libs/tex/texturing.h:46     -> b2tex_prepare_mesh (resident API)
 *
 * Plain pointers and sizes only; host buffers are owned by the caller, device memory by the
 * library.  Every function returns 0 on success and a non-zero status otherwise;
 * b2tex_last_error() returns a thread-local message (the C++ veneer turns it into the
 * std::runtime_error the reference throws, calculate_data_costs.cpp:315-318,
 * view_selection.cpp:126-128).  There is no CPU fallback: without a CUDA device every entry
 * point fails with B2TEX_ERR_CUDA.
 */
#ifndef B2TEX_H
#define B2TEX_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2TEX_OK 0
#define B2TEX_ERR_CUDA 1      /* CUDA runtime error / no device */
#define B2TEX_ERR_LIMITS 2    /* "Exeeded maximal number of faces/views" (calculate_data_costs.cpp:315-318) */
#define B2TEX_ERR_ARG 3       /* bad argument / stage prerequisites missing */
#define B2TEX_ERR_LABELING 4  /* "Incorrect labeling" (view_selection.cpp:126-128) */
#define B2TEX_ERR_UNSUPPORTED 5

/* tex::TextureView camera + image (libs/tex/texture_view.h:39-52) as POD */
typedef struct {
    float pos[3];        /* camera centre, world */
    float viewdir[3];    /* viewing direction, world */
    float proj[9];       /* calibration, row major 3x3 (pixels) */
    float w2c[16];       /* world_to_cam, row major 4x4 */
    int32_t width, height;
    const uint8_t *rgb;  /* H x W x 3 interleaved, host memory */
} b2tex_view;

/* the fields of tex::Settings the path reads (libs/tex/settings.h:82-94) */
typedef struct {
    int32_t data_term;                 /* 0 DATA_TERM_AREA, 1 DATA_TERM_GMI */
    int32_t outlier_removal;           /* 0 NONE, 1 GAUSS_DAMPING, 2 GAUSS_CLAMPING (settings.h:70-74) */
    int32_t geometric_visibility_test; /* bool */
} b2tex_settings;

typedef struct {
    uint64_t nnz;          /* DataCosts entries */
    uint64_t candidates;   /* (face,view) pairs that passed culling + projection */
    uint64_t rays;         /* distinct (vertex,view) visibility rays traced */
    float max_quality;     /* calculate_data_costs.cpp:304 */
    float percentile;      /* calculate_data_costs.cpp:305 */
} b2tex_dc_info;

/* mapMAP control as configured at view_selection.cpp:84,103-115, mapped onto the forest-BCD solver */
typedef struct {
    uint32_t max_iterations;
    uint32_t rounds;       /* forest growth rounds per iteration */
    uint32_t root_div;     /* one root candidate per root_div nodes; 0 = single root */
    uint32_t seed;         /* initial_seed */
    uint32_t window;       /* StopWhenReturnsDiminish(window, ratio) */
    float ratio;
    uint32_t num_parts;    /* logical face partitions (>=1); >1 reproduces the multi-GPU schedule */
    uint32_t num_views;    /* DataCosts::rows() for the one-shot call; 0 = derive from the entries */
    uint32_t use_multilevel;   /* mapMAP_control::use_multilevel: after the stop rule fires, contract every same-label
                                  region into one node, solve the contracted MRF (weighted Potts) from the current labels
                                  and go back to the faces while that lowers the energy.  One GPU, whole mesh, num_parts 1
                                  only (else B2TEX_ERR_UNSUPPORTED).  Default 0. */
    uint32_t use_spanning_tree;   /* mapMAP_control::use_spanning_tree: before the iterations on induced forests, a phase of
                                     iterations on spanning forests of the seen faces (BFS from the same roots, every
                                     non-tree neighbour fixed at its label from the start of the iteration; an iteration
                                     that raises the energy is undone), until the stop rule fires.  The induced-forest
                                     phase follows with the window restarted, then the multilevel schedule if
                                     use_multilevel.  One GPU, whole mesh, num_parts 1 only (else B2TEX_ERR_UNSUPPORTED).
                                     Default 0. */
    uint32_t spanning_tree_multilevel_after_n_iterations;   /* mapMAP_control's field of that name (n): with n > 0,
                                     a multilevel step (contract the labeling, one spanning-tree iteration on the contracted
                                     MRF with weighted Potts terms, undone if it raises the energy) follows every n-th
                                     iteration of the spanning phase, unless the stop rule has fired or max_iterations is
                                     reached.  The induced-forest phase follows and is the last one: the post-acyclic
                                     multilevel schedule does not run.  n > 0 needs use_spanning_tree = 1 and
                                     use_multilevel = 1 (else B2TEX_ERR_ARG).  Default 0. */
} b2tex_mrf_params;

typedef struct {
    uint32_t iterations;
    double energy_initial;
    double energy_final;
    uint64_t unseen;       /* "faces have not been seen" view_selection.cpp:132 */
    uint64_t sweep_bytes;  /* algorithmic bytes of one sweep (SURVEY 8d): 14 nnz + 20 F */
    uint32_t multilevel_passes;   /* use_multilevel: contractions whose coarse solve lowered the energy */
    uint32_t coarse_nodes;        /* use_multilevel: nodes of the last contraction */
    uint32_t spanning_tree_iterations;   /* use_spanning_tree: iterations of the spanning phase (numbered 1 ..) */
    uint32_t spanning_tree_rejected;     /* use_spanning_tree: of those, the ones that were undone */
    /* how the tree solver (k_tree) ran, fixed per run from the input */
    uint32_t tree_group;         /* lanes per tree node: 4, 8, 16 or 32, from the candidates per face */
    uint32_t tree_cap;           /* longest label list the shared-memory scratch holds; trees with a longer list are
                                    solved through global memory */
    uint32_t label_mask_words;   /* 32-bit words of the per-node label bitmask (0: more than 2047 views, labels found
                                    by bisection of the sorted list) */
    uint32_t global_trees;       /* trees solved through global memory (a node of degree > 3 or a label list longer
                                    than tree_cap), summed over all iterations and phases */
    uint32_t multilevel_steps;            /* spanning_tree_multilevel_after_n_iterations > 0: multilevel steps of the
                                             spanning phase (counted in spanning_tree_iterations, which numbers both) */
    uint32_t multilevel_steps_rejected;   /* of those, the ones that were undone (not in spanning_tree_rejected) */
} b2tex_mrf_info;

typedef struct {
    uint32_t num_rows;       /* Lhs dimensionality, global_seam_leveling.cpp:253 */
    uint32_t num_a_rows;
    uint32_t num_gamma_rows;
    uint64_t nnz_full;       /* non-zeros of the full symmetric Lhs */
    uint32_t iterations[3];  /* cg.iterations() per colour channel, :280 */
    float residual[3];       /* cg.error() per colour channel, :281 */
    uint32_t cg_launch_iterations; /* iterations executed by the batched kernel = max over channels */
    float cg_ms;             /* device time of the PCG kernel (CUDA events) */
} b2tex_seam_info;

typedef struct {
    uint32_t num_patches;   /* "texture patches." generate_texture_patches.cpp:597 (seen faces only) */
    uint32_t num_faces;     /* faces with a label != 0 = sum of the patches' face counts */
    uint64_t num_pixels;    /* sum of width * height over the patches */
} b2tex_patch_info;

typedef struct {
    uint32_t num_seam_edges;    /* find_seam_edges, seam_leveling.cpp:16-59 */
    uint32_t num_edge_samples;  /* sum of ceil(2 * max projected length), local_seam_leveling.cpp:139 */
    uint32_t num_vertices;      /* vertices projected into more than one patch, :157 */
    uint32_t num_unknowns;      /* blending mask == 255 pixels of all patches (interior of the 20 px strips) */
    uint32_t iterations[3];     /* CG iterations per colour channel (one batched solve for all patches) */
    float residual[3];          /* |r| / |b| per colour channel at exit */
} b2tex_local_seam_info;

/* radial distortion of one view: line 2 of its MVE .cam file (generate_texture_views.cpp:138-146) */
typedef struct {
    float flen;      /* focal length normalised by the larger image side */
    float dist[2];   /* dist[0] == 0: no distortion; dist[1] != 0: Bundler k2 k4 model; else VisualSFM with k = dist[0] */
} b2tex_distortion;

/* sizes of the mesh graph b2tex_build_mesh_graph derives */
typedef struct {
    uint32_t num_adjacency;          /* adj_ptr[F]: directed face-adjacency entries */
    uint32_t num_vertex_faces;       /* vf_ptr[Vn] */
    uint32_t num_vertex_neighbours;  /* vv_ptr[Vn] */
    uint32_t max_face_degree;        /* longest adjacency row */
    uint32_t num_non_manifold_edges; /* undirected edges shared by more than two faces */
} b2tex_graph_info;

/* what b2tex_prepare_mesh did */
typedef struct {
    uint32_t num_faces_in;       /* faces passed in */
    uint32_t num_faces;          /* faces kept (F of the context afterwards) */
    uint32_t num_redundant;      /* "Removed N redundant faces." (prepare_mesh.cpp:60) */
    uint32_t num_zero_normals;   /* kept faces whose normal is 0 */
    b2tex_graph_info graph;      /* what b2tex_build_mesh_graph reports for the kept faces */
} b2tex_mesh_prep_info;

typedef struct b2tex_ctx b2tex_ctx;

/* ---- lifetime ---- */
int b2tex_create(int device, b2tex_ctx **out);
void b2tex_destroy(b2tex_ctx *ctx);
const char *b2tex_last_error(void);
void b2tex_free(void *host_ptr);                 /* frees buffers returned by one-shot calls */
int b2tex_device_synchronize(b2tex_ctx *ctx);
uint64_t b2tex_stream(b2tex_ctx *ctx);            /* the cudaStream_t every kernel is launched on */
uint64_t b2tex_launch_count(void);                /* kernels of this library launched by this process so far (CUB's not counted) */
/* per-kernel CUDA-event timing: enable, run stages, read "name ms algorithmic_bytes" lines */
int b2tex_profile(b2tex_ctx *ctx, int enable);
int b2tex_profile_report(b2tex_ctx *ctx, char *buf, uint64_t cap);
void b2tex_default_mrf_params(b2tex_mrf_params *p);
/* the defaults with mapMAP's control as texrecon sets it (view_selection.cpp:103-115): use_spanning_tree = 1,
 * use_multilevel = 1, spanning_tree_multilevel_after_n_iterations = 5 */
void b2tex_texrecon_mrf_params(b2tex_mrf_params *p);

/* ---- resident API: upload once, run stages on the device, download results ----
 *
 * A context holds uploads and the results derived from them.  An item stays valid until one it is derived from changes
 * (transitively); a stage, or a download, whose inputs are not valid returns B2TEX_ERR_ARG and names them.
 *
 *   item             made valid by                                          derived from
 *   mesh             set_mesh, prepare_mesh                                 -
 *   prepared mesh    prepare_mesh (vertex normals, kept face ids)           mesh
 *   BVH              the data-cost stage                                    mesh
 *   face adjacency   set_adjacency, build_mesh_graph, prepare_mesh          mesh
 *   vertex rings     set_vertex_rings, build_mesh_graph, prepare_mesh       mesh
 *   views            set_views (cameras, number of views)                   -
 *   pixels           set_views, undistort_views                             views
 *   prepared images  the stages that read pixels                            pixels
 *   data costs       data_costs_run / _normalize, set_data_costs            mesh, pixels; set_face_range invalidates them
 *   view selection   mrf_init, view_selection_run (the state mrf_iterate,   data costs, face adjacency
 *     state          mrf_energy and mrf_sample_forest read)
 *   labels           set_labels, mrf_init, mrf_iterate, view_selection_run  mesh, views
 *   seam system      seam_run, seam_assemble                                mesh, pixels, vertex rings, labels
 *   seam solution    seam_run, seam_mg_solve                                seam system
 *   texture patches  texture_patches_run                                    mesh, pixels, face adjacency, labels
 *
 * A stage invalidates its own result when it starts and marks it valid only when it succeeds. */
int b2tex_set_mesh(b2tex_ctx *ctx, const float *verts, uint32_t num_verts, const uint32_t *faces,
                   const float *face_normals, uint32_t num_faces);
int b2tex_set_views(b2tex_ctx *ctx, const b2tex_view *views, uint32_t num_views);
int b2tex_set_adjacency(b2tex_ctx *ctx, const uint32_t *adj_ptr, const uint32_t *adj_idx);
int b2tex_set_vertex_rings(b2tex_ctx *ctx, const uint32_t *vf_ptr, const uint32_t *vf_idx,
                           const uint32_t *vv_ptr, const uint32_t *vv_idx);
/* Derives the face adjacency (build_adjacency_graph.cpp:16-53) and the vertex rings from the mesh set by b2tex_set_mesh,
 * on the device; afterwards the context is as if b2tex_set_adjacency and b2tex_set_vertex_rings had been called with the
 * arrays scene.face_adjacency / scene.vertex_rings give: adjacency rows hold the lower neighbours ascending, then the
 * higher ones by the slot of the shared edge and ascending, each face once; vf rows the incident faces ascending (a face
 * with a repeated vertex twice); vv rows the distinct u of the directed edges (v, u) ascending.  B2TEX_ERR_ARG without a
 * mesh or with a face index >= num_verts (the first such face is named); B2TEX_ERR_LIMITS when a count does not fit the
 * 32-bit offsets.  A failed build leaves the context without a graph.  info may be NULL. */
int b2tex_build_mesh_graph(b2tex_ctx *ctx, b2tex_graph_info *info);
/* the resident graph (derived or uploaded); arrays sized from b2tex_graph_info: adj_ptr[F+1], adj_idx[num_adjacency],
 * vf_ptr[Vn+1], vf_idx[num_vertex_faces], vv_ptr[Vn+1], vv_idx[num_vertex_neighbours]; any pointer may be NULL;
 * B2TEX_ERR_ARG when a requested part is not resident */
int b2tex_mesh_graph_download(b2tex_ctx *ctx, uint32_t *adj_ptr, uint32_t *adj_idx, uint32_t *vf_ptr, uint32_t *vf_idx,
                              uint32_t *vv_ptr, uint32_t *vv_idx);
/* tex::prepare_mesh (prepare_mesh.cpp:14-70) on the raw mesh, as texrecon loads it: face i is dropped when a face j > i has
 * all its vertices among those of i (exact duplicates in any order keep the highest id; a proper triangle also goes when a
 * later degenerate face such as (a, a, b) uses only its vertices), the kept faces stay in their order, the vertices are
 * untouched.  Then the face normals of the kept faces (normalised cross(b - a, c - a), 0 when its length is 0), the mesh
 * graph (b2tex_build_mesh_graph) and angle-weighted vertex normals.  Afterwards the context is exactly as after
 * b2tex_set_mesh(verts, kept faces, their normals) + b2tex_build_mesh_graph, with the vertex normals resident.
 * B2TEX_ERR_ARG for NULL pointers, num_faces == 0 or a face index >= num_verts (the first
 * such face is named); B2TEX_ERR_LIMITS when a count does not fit the 32-bit offsets.  A failure leaves no mesh.  info may
 * be NULL. */
int b2tex_prepare_mesh(b2tex_ctx *ctx, const float *verts, uint32_t num_verts, const uint32_t *faces,
                       uint32_t num_faces, b2tex_mesh_prep_info *info);
/* faces[F'][3], face_normals[F'][3], vertex_normals[Vn][3], kept_face_ids[F'] (old id of each kept face); any may be NULL.
 * B2TEX_ERR_ARG unless the last b2tex_prepare_mesh / b2tex_set_mesh on this context was a successful prepare. */
int b2tex_prepared_mesh_download(b2tex_ctx *ctx, uint32_t *faces, float *face_normals, float *vertex_normals,
                                 uint32_t *kept_face_ids);
int b2tex_set_data_costs(b2tex_ctx *ctx, const uint64_t *face_ptr, const uint16_t *view,
                         const float *cost);
int b2tex_set_labels(b2tex_ctx *ctx, const uint32_t *labels);
/* restrict this context to faces [face_begin, face_end) for the data-cost stage (multi-GPU shard);
 * default is all faces */
int b2tex_set_face_range(b2tex_ctx *ctx, uint32_t face_begin, uint32_t face_end);
/* Undistorts the resident images in place, as the reference does while it loads a .cam scene
 * (generate_texture_views.cpp:154-162, MVE image_undistort_k2k4 / image_undistort_vsfm): every later stage reads the
 * undistorted pixels.  d[num_views], num_views == the number of views set.  Views with dist[0] == 0 stay untouched;
 * pixels whose source falls outside the image become 0 (and so may give the view a validity mask).  B2TEX_ERR_ARG if no
 * views are set, num_views differs, or a view to undistort has a focal length that is not finite and positive.  Call it
 * after b2tex_set_views and before the stages. */
int b2tex_undistort_views(b2tex_ctx *ctx, const b2tex_distortion *d, uint32_t num_views);

int b2tex_data_costs_run(b2tex_ctx *ctx, const b2tex_settings *settings, b2tex_dc_info *info);
/* split form of the normalisation for sharded runs (calculate_data_costs.cpp:277-302):
 * qualities -> [allreduce max] -> histogram -> [allreduce sum] -> normalise */
int b2tex_data_costs_qualities(b2tex_ctx *ctx, const b2tex_settings *settings, b2tex_dc_info *info);
int b2tex_data_costs_histogram(b2tex_ctx *ctx, float global_max, uint32_t *bins10000_device_or_host,
                               int to_host);
int b2tex_data_costs_normalize(b2tex_ctx *ctx, float global_max, const uint32_t *bins10000_host,
                               b2tex_dc_info *info);
int b2tex_data_costs_download(b2tex_ctx *ctx, uint64_t *face_ptr, uint16_t *view, float *cost,
                              float *quality_or_null);

int b2tex_view_selection_run(b2tex_ctx *ctx, const b2tex_mrf_params *params, b2tex_mrf_info *info,
                             double *energy_trace_or_null);
/* optional: performs every device allocation b2tex_view_selection_run(params) will need and nothing else.  Only a caller
 * that drives several peer ranks from ONE process needs it (all ranks prepare before the first one runs: cudaMalloc waits
 * for the whole device, which a rank already spinning in a cross-rank barrier kernel would block for good). */
int b2tex_view_selection_prepare(b2tex_ctx *ctx, const b2tex_mrf_params *params);
int b2tex_labels_download(b2tex_ctx *ctx, uint32_t *labels);
/* Multi-GPU view selection (one process per GPU, at most 8): rank r owns the faces [r * ceil(F / P), (r + 1) * ceil(F / P))
 * (b2tex_set_face_range) and runs b2tex_view_selection_run with params->num_parts = P like a single GPU would.  Before
 * that, once per mesh size: every rank calls b2tex_mrf_mg_export (allocates a peer-visible block holding its full-length
 * label array, the energy slots and the barrier flags; the context's labels live inside it from then on), the 64-byte
 * cudaIpc handles are exchanged by the caller (e.g. one all-gather over torch.distributed) and imported with
 * b2tex_mrf_mg_import.  Inside the run the ranks exchange only the labels of their boundary faces -- stored straight
 * into the label arrays of the ranks that own a neighbouring face -- and their partial energies, through NVLink peer
 * memory with epoch-flag barriers; every rank takes the identical stop decision (view_selection.cpp:84) from the
 * identical fixed-point sum.  No NCCL call and no host round trip per iteration. */
int b2tex_mrf_mg_export(b2tex_ctx *ctx, uint32_t rank, uint32_t num_ranks, void *ipc_handle_64_bytes);
int b2tex_mrf_mg_import(b2tex_ctx *ctx, uint32_t peer_rank, const void *ipc_handle_64_bytes);
/* Peers that live in the SAME process (several contexts driven by threads) cannot open each other's IPC handles: after
 * the export they attach the raw device pointer of the peer's block instead.  which: 0 = view selection block
 * (b2tex_mrf_mg_export), 1 = seam solve block (b2tex_seam_mg_export). */
uint64_t b2tex_peer_block(b2tex_ctx *ctx, int which);
int b2tex_peer_attach(b2tex_ctx *ctx, int which, uint32_t peer_rank, uint64_t peer_block_device_ptr);
/* building blocks of one solver iteration, exposed so that a sharded run can exchange boundary
 * labels between iterations (SURVEY 8e); view_selection_run = init + loop(iterate, energy) */
int b2tex_mrf_init(b2tex_ctx *ctx, const b2tex_mrf_params *params, int64_t *energy_fixed);
int b2tex_mrf_iterate(b2tex_ctx *ctx, uint32_t iteration, int64_t *energy_fixed);
/* energy of the owned faces under the labels currently on the device (call after a label exchange) */
int b2tex_mrf_energy(b2tex_ctx *ctx, int64_t *energy_fixed);
int b2tex_mrf_sample_forest(b2tex_ctx *ctx, const b2tex_mrf_params *params, uint32_t iteration,
                            uint32_t *level_out_host);

int b2tex_seam_run(b2tex_ctx *ctx, b2tex_seam_info *info);
/* Multi-GPU solve of the same system (one process per GPU): every rank assembles (b2tex_seam_assemble = b2tex_seam_run
 * without the PCG), allocates a peer-visible exchange block and exports its 64-byte cudaIpc handle, imports the handles
 * of all peers (exchanged by the caller, e.g. an all-gather over torch.distributed), then every rank calls
 * b2tex_seam_mg_solve: one persistent cooperative kernel per GPU that runs the PCG on its slice of the rows and exchanges
 * the search direction and the dot products with its peers through NVLink peer memory inside the kernel.  Every rank ends
 * with the complete solution (b2tex_seam_download).  At most 8 ranks. */
int b2tex_seam_assemble(b2tex_ctx *ctx, b2tex_seam_info *info);
int b2tex_seam_mg_export(b2tex_ctx *ctx, uint32_t rank, uint32_t num_ranks, void *ipc_handle_64_bytes);
int b2tex_seam_mg_import(b2tex_ctx *ctx, uint32_t peer_rank, const void *ipc_handle_64_bytes);
int b2tex_seam_mg_solve(b2tex_ctx *ctx, b2tex_seam_info *info);
int b2tex_seam_download(b2tex_ctx *ctx, uint32_t *row_ptr, uint32_t *row_label, float *x,
                        float *rhs_or_null);
/* full symmetric CSR of Lhs (for tests / inspection); arrays sized from b2tex_seam_info */
int b2tex_seam_matrix_download(b2tex_ctx *ctx, uint32_t *csr_ptr, uint32_t *csr_col, float *csr_val);
/* tex::generate_texture_patches for the seen faces (generate_texture_patches.cpp:78-138,453-538; hole filling
 * :140-451 is not built: faces with label 0 get no patch) followed by TexturePatch::adjust_colors per patch
 * (texture_patch.cpp:41-116) with the solved offsets (apply_adjust = 1, global_seam_leveling.cpp:293-323; needs
 * b2tex_seam_run) or with zeros (apply_adjust = 0, texrecon.cpp:174-183).  Needs mesh, views, adjacency, labels.
 * Patch ids follow ascending labels (the reference's ids depend on OpenMP scheduling, :469,514-518). */
int b2tex_texture_patches_run(b2tex_ctx *ctx, int apply_adjust, b2tex_patch_info *info);
/* desc[num_patches][8] = label, min_x, min_y (view pixel of patch pixel (0,0)), width, height, first face slot,
 * number of faces, 0; faces[num_faces]; texcoords[num_faces][3][2]; per pixel (patch after patch, row major):
 * images[num_pixels][3] float, validity[num_pixels], blending[num_pixels] (255 inside, 64 within sqrt(2), 0).
 * Any pointer may be NULL. */
int b2tex_texture_patches_download(b2tex_ctx *ctx, int32_t *desc, uint32_t *faces, float *texcoords, float *images,
                                   uint8_t *validity, uint8_t *blending);
/* tex::local_seam_leveling (local_seam_leveling.cpp:105-204) on the patches b2tex_texture_patches_run left on the device:
 * mean colours along the seam edges and at shared vertices are stamped into every adjacent patch, the blending mask keeps
 * a 20 pixel strip (TexturePatch::prepare_blending_mask), the strip is Poisson-blended towards the stamped colours
 * (poisson_blend, alpha = 1; one batched CG over all patches instead of one SparseLU per patch: same linear systems,
 * agreement to the CG tolerance) and pixels outside the patch boundary are invalidated (TexturePatch::blend).
 * Download the result with b2tex_texture_patches_download (the blending mask is the one used for blending; the
 * reference releases it at :201). */
int b2tex_local_seam_leveling_run(b2tex_ctx *ctx, b2tex_local_seam_info *info);
/* raw device pointers of resident results (torch / NCCL plumbing); 0 if absent */
uint64_t b2tex_device_ptr(b2tex_ctx *ctx, const char *name, uint64_t *num_elements);

/* ---- one-shot host-buffer entry points (what the reference-side binding calls) ----
 * They run on the calling thread's current CUDA device (cudaGetDevice) and keep up to two finished contexts (stream +
 * device buffers) cached for the next call; b2tex_release_cached_contexts() frees them. */
void b2tex_release_cached_contexts(void);
/* tex::calculate_data_costs: out arrays are malloc'ed by the library (b2tex_free), CSR by face:
 * face_ptr[F+1], view[nnz] ascending per face, cost[nnz]. */
int b2tex_calculate_data_costs(const float *verts, uint32_t num_verts, const uint32_t *faces,
                               const float *face_normals, uint32_t num_faces,
                               const b2tex_view *views, uint32_t num_views,
                               const b2tex_settings *settings, uint64_t **face_ptr_out,
                               uint16_t **view_out, float **cost_out, b2tex_dc_info *info);
/* same, into caller-owned (ideally pinned) buffers of `capacity` entries: no allocation, no extra copy;
 * fails with B2TEX_ERR_ARG (info->nnz = required size) when the capacity is too small */
int b2tex_calculate_data_costs_into(const float *verts, uint32_t num_verts, const uint32_t *faces,
                                    const float *face_normals, uint32_t num_faces,
                                    const b2tex_view *views, uint32_t num_views,
                                    const b2tex_settings *settings, uint64_t *face_ptr, uint16_t *view,
                                    float *cost, uint64_t capacity, b2tex_dc_info *info);
/* tex::postprocess_face_infos (libs/tex/texturing.h:71-74, calculate_data_costs.cpp:253-306) for qualities the caller
 * computed: per face (CSR face_ptr[F+1]) the infos in ascending view order -- view[n], quality[n] and, with outlier
 * removal, the mean YCbCr colour mean_color_ycbcr[n][3] (NULL otherwise).  Photometric outlier removal, quality == 0
 * entries dropped, 99.5 % percentile of the 10 000-bin histogram, cost = 1 - min(1, quality / percentile).  Out arrays are
 * caller allocated: face_ptr_out[F+1], view_out / cost_out with room for n entries. */
int b2tex_postprocess_face_infos(uint32_t num_faces, const uint64_t *face_ptr, const uint16_t *view, const float *quality,
                                 const float *mean_color_ycbcr, const b2tex_settings *settings, uint64_t *face_ptr_out,
                                 uint16_t *view_out, float *cost_out, b2tex_dc_info *info);
/* tex::view_selection: labels_out[F] (0 = unseen, else view index + 1) */
int b2tex_view_selection(uint32_t num_faces, const uint32_t *adj_ptr, const uint32_t *adj_idx,
                         const uint64_t *face_ptr, const uint16_t *view, const float *cost,
                         const b2tex_mrf_params *params_or_null, uint32_t *labels_out,
                         b2tex_mrf_info *info);
/* tex::global_seam_leveling up to the per-(vertex,label) adjust values (:283-289):
 * row_ptr_out[Vn+1] caller allocated; row_label/x (R and R*3, centred) malloc'ed by the library.
 * vf_ptr, vf_idx, vv_ptr and vv_idx all NULL: the rings are derived from the mesh on the device (b2tex_build_mesh_graph);
 * some NULL and some not: B2TEX_ERR_ARG. */
int b2tex_global_seam_leveling(const float *verts, uint32_t num_verts, const uint32_t *faces,
                               uint32_t num_faces, const uint32_t *vf_ptr, const uint32_t *vf_idx,
                               const uint32_t *vv_ptr, const uint32_t *vv_idx,
                               const uint32_t *labels, const b2tex_view *views, uint32_t num_views,
                               uint32_t *row_ptr_out, uint32_t **row_label_out, float **x_out,
                               b2tex_seam_info *info);

/* The three stages back to back on one upload -- what texrecon does between texrecon.cpp:100 and :171
 * when it writes no intermediate results (--no_intermediate_results, arguments.cpp:88-89): the mesh and
 * the images cross PCIe once, DataCosts stay on the device, only labels[F] and the per-(vertex,label)
 * adjust values come back.  Optional outputs may be NULL.  row_label/x are malloc'ed (b2tex_free).
 * The six topology arrays (adj_ptr .. vv_idx) all NULL: the graph is derived from the mesh on the device
 * (b2tex_build_mesh_graph); some NULL and some not: B2TEX_ERR_ARG. */
int b2tex_texture_hot_path(const float *verts, uint32_t num_verts, const uint32_t *faces,
                           const float *face_normals, uint32_t num_faces, const b2tex_view *views,
                           uint32_t num_views, const uint32_t *adj_ptr, const uint32_t *adj_idx,
                           const uint32_t *vf_ptr, const uint32_t *vf_idx, const uint32_t *vv_ptr,
                           const uint32_t *vv_idx, const b2tex_settings *settings,
                           const b2tex_mrf_params *mrf_params_or_null, uint32_t *labels_out,
                           uint32_t *row_ptr_out, uint32_t **row_label_out, float **x_out,
                           b2tex_dc_info *dc_info, b2tex_mrf_info *mrf_info, b2tex_seam_info *seam_info);

/* Everything texrecon does between texrecon.cpp:160 and :189 on one upload: texture patches for the seen faces,
 * global seam leveling (do_global; else the zero-offset validity pass of :174-183), local seam leveling (do_local).
 * Outputs are malloc'ed (b2tex_free) and laid out as b2tex_texture_patches_download describes; info structs may be NULL.
 * The six topology arrays (adj_ptr .. vv_idx) all NULL: the graph is derived from the mesh on the device
 * (b2tex_build_mesh_graph); some NULL and some not: B2TEX_ERR_ARG. */
int b2tex_seam_leveling_patches(const float *verts, uint32_t num_verts, const uint32_t *faces, uint32_t num_faces,
                                const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint32_t *vf_ptr,
                                const uint32_t *vf_idx, const uint32_t *vv_ptr, const uint32_t *vv_idx,
                                const uint32_t *labels, const b2tex_view *views, uint32_t num_views, int do_global,
                                int do_local, int32_t **desc_out, uint32_t **faces_out, float **texcoords_out,
                                float **images_out, uint8_t **validity_out, b2tex_patch_info *patch_info,
                                b2tex_seam_info *seam_info, b2tex_local_seam_info *local_info);

#ifdef __cplusplus
}
#endif
#endif /* B2TEX_H */
