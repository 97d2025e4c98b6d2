// common.cuh -- context, device buffers and error plumbing shared by the sm_90a kernels.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>

#include "../../include/b2tex.h"
#include "state.h"

namespace b2 {

void set_error(const char *fmt, ...);
// every launch of one of this library's kernels is counted (process wide): `B2_LAUNCH kernel<<<...>>>(...)`
void count_launch();
#define B2_LAUNCH b2::count_launch(),

#define B2_CUDA(expr)                                                                         \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess) {                                                              \
            b2::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return B2TEX_ERR_CUDA;                                                            \
        }                                                                                     \
    } while (0)

#define B2_TRY(expr)                    \
    do {                                \
        int _rc = (expr);               \
        if (_rc != B2TEX_OK) return _rc; \
    } while (0)

#define B2_KERNEL_CHECK() B2_CUDA(cudaGetLastError())

template <typename T>
struct DevBuf {
    T *p = nullptr;
    size_t n = 0;    // elements in use
    size_t cap = 0;  // elements allocated
    bool borrowed = false;  // p points into memory somebody else owns (a peer-visible block): never freed, never grown
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { release(); }
    void release()
    {
        if (p && !borrowed) cudaFree(p);
        p = nullptr;
        n = cap = 0;
        borrowed = false;
    }
    // use `count` elements at `ptr` (owned by the caller) as this buffer
    void borrow(T *ptr, size_t count)
    {
        release();
        p = ptr; n = cap = count; borrowed = true;
    }
    // grow-only allocation; contents are NOT preserved
    int alloc(size_t count)
    {
        if (count > cap) {
            if (borrowed) { set_error("a peer-mapped buffer cannot grow (%zu > %zu elements)", count, cap); return B2TEX_ERR_ARG; }
            if (p) cudaFree(p);
            p = nullptr;
            cap = 0;
            size_t want = count ? count : 1;
            // 64 bytes of slack: 16-byte-granular bulk copies (cp.async.bulk) may read past the last element
            cudaError_t e = cudaMalloc((void **)&p, want * sizeof(T) + 64);
            if (e != cudaSuccess) {
                set_error("cudaMalloc(%zu bytes) failed: %s", want * sizeof(T), cudaGetErrorString(e));
                n = 0;
                return B2TEX_ERR_CUDA;
            }
            cap = want;
        }
        n = count;
        return B2TEX_OK;
    }
    int upload(const T *host, size_t count, cudaStream_t s)
    {
        B2_TRY(alloc(count));
        if (count) B2_CUDA(cudaMemcpyAsync(p, host, count * sizeof(T), cudaMemcpyHostToDevice, s));
        return B2TEX_OK;
    }
    int download(T *host, size_t count, cudaStream_t s) const
    {
        if (count) B2_CUDA(cudaMemcpyAsync(host, p, count * sizeof(T), cudaMemcpyDeviceToHost, s));
        return B2TEX_OK;
    }
    int zero(cudaStream_t s)
    {
        if (n) B2_CUDA(cudaMemsetAsync(p, 0, n * sizeof(T), s));
        return B2TEX_OK;
    }
};

// device-side copy of one view (camera + prepared images)
struct ViewDev {
    float pos[3];
    float dir[3];
    float proj[9];
    float w2c[12];
    int32_t w, h;
    const uint8_t *rgb;    // H*W*3
    const uint8_t *grad;   // H*W (null for DATA_TERM_AREA)
    const uint8_t *valid4; // H*W, 1 = all four bilinear taps valid; null = everything valid
};

// two-child BVH node: both child boxes in one 64-byte record
struct __align__(16) BvhNode {
    float lo0[3], hi0[3];  // left child box
    float lo1[3], hi1[3];  // right child box
    int32_t left, right;   // >=0 internal node index, <0: ~(sorted triangle slot)
    int32_t pad0, pad1;
};

struct Bvh {
    DevBuf<BvhNode> nodes;      // N-1 internal nodes (N>=2)
    DevBuf<float> tri;          // 9 floats per triangle in Morton order
    uint32_t num_tris = 0;
};

}  // namespace b2

namespace b2 {
struct KTimer {
    const char *name;
    cudaEvent_t a, b;
    double bytes;  // algorithmic bytes of this launch (0 = not accounted)
};
}  // namespace b2

namespace b2 { struct PatchState; }  // texture patches (patches.cu)
namespace b2 { struct MgState; }     // multi-GPU seam solve (seam_mg.cu)
namespace b2 { struct MrfMgState; }  // multi-GPU view selection: peer-visible labels + energy slots (mrf.cu)

// The opaque C-ABI context.
struct b2tex_ctx {
    bool profile = false;
    std::vector<b2::KTimer> timers;

    int device = 0;
    int num_sms = 0;
    cudaStream_t stream = nullptr;
    // one-shot entry points: the image upload runs on its own stream while the stages that need no pixels (BVH, cull,
    // visibility rays) already run; `images_uploaded` is what the first pixel consumer waits for
    b2::DevBuf<uint8_t> tmap_dev;   // the TMA descriptor of the rgb images (128 B) + a timeout counter
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t images_uploaded = nullptr;
    bool defer_image_sync = false, images_in_flight = false;
    bool any_corner_flag = false;   // some view has a zero-sum corner pixel: validity masks exist and the cull reads them
    uint32_t valid = 0;             // the items (state.h) that are up to date: invalidate / mark_valid / require below

    // mesh
    uint32_t Vn = 0, F = 0;
    uint32_t face_begin = 0, face_end = 0;
    b2::DevBuf<float> verts, normals;
    b2::DevBuf<uint32_t> faces;
    // prepare_mesh (prepare.cu): vertex normals [3 Vn] and the input id of every kept face [F]
    b2::DevBuf<float> vnormals;
    b2::DevBuf<uint32_t> kept_ids;

    // views
    uint32_t K = 0;
    std::vector<b2tex_view> views_host;   // camera params (rgb pointer = caller memory, not kept)
    b2::DevBuf<uint8_t> rgb, grad, valid4;
    std::vector<size_t> img_off;          // pixel offset of each view in grad/valid4 (rgb: *3)
    b2::DevBuf<b2::ViewDev> views_dev;
    int prepared_data_term = -1;          // the data term of the prepared images (while IMAGES is valid)

    // bvh
    b2::Bvh bvh;
    b2::DevBuf<uint32_t> vrank, vorder;  // Morton rank of every vertex and its inverse
    // persistent scratch (grow only): cudaMalloc/cudaFree inside a stage would serialise the device
    b2::DevBuf<uint32_t> s_bnd, s_ids_in, s_ids_out, s_counters, s_vi_in, s_cnt32, s_row_vertex, s_rcnt, s_pass_bits, s_limits;
    b2::DevBuf<uint64_t> s_keys_in, s_keys_out, s_vk_in, s_vk_out, s_cnt64;
    b2::DevBuf<int> s_parent_internal, s_parent_leaf;

    // data costs (CSR by face over [face_begin, face_end) -> global face ids keep absolute ptr layout)
    b2::DevBuf<uint64_t> dc_ptr;       // F+1
    b2::DevBuf<uint16_t> dc_view;      // nnz
    b2::DevBuf<float> dc_cost;         // nnz
    b2::DevBuf<float> dc_quality;      // nnz
    uint64_t nnz = 0;
    // scratch of the data-cost stage
    b2::DevBuf<uint64_t> cand_ptr;     // F+1
    b2::DevBuf<uint16_t> cand_view;
    b2::DevBuf<uint32_t> cand_face;
    b2::DevBuf<float> cand_q, cand_ycc;   // cand_ycc: mean YCbCr per candidate (outlier removal only)
    b2::DevBuf<uint8_t> cand_flag;
    b2::DevBuf<uint32_t> need_bits, occ_bits;
    b2::DevBuf<uint32_t> hist;         // 10000 bins
    b2::DevBuf<uint32_t> scalars;      // misc device scalars
    b2::DevBuf<uint8_t> cub_tmp;
    uint64_t num_cand = 0;

    // graph + labels
    b2::DevBuf<uint32_t> adj_ptr, adj_idx;
    b2::DevBuf<uint32_t> labels;

    // mrf scratch
    b2::DevBuf<float> mrf_H, mrf_hminp1;    // global-memory DP tables (trees that do not fit in shared memory only)
    b2::DevBuf<uint32_t> mrf_amin, mrf_level, mrf_order, mrf_ctl, mrf_state;
    b2::DevBuf<uint32_t> mrf_lidx;          // position of every node's label in its label list
    b2::DevBuf<uint16_t> mrf_olev;          // level of order[i]
    b2::DevBuf<uint32_t> mrf_pos;           // position of a node in order (forest nodes), else 0xFFFFFFFF
    b2::DevBuf<uint2> mrf_tjoin;            // per node (tree, arrival number)
    b2::DevBuf<uint4> mrf_ttab;             // per tree (nodes, labels, first order index, flags)
    b2::DevBuf<unsigned long long> mrf_energy;   // [max_iterations + 2] fixed-point energies
    b2::DevBuf<unsigned long long> mrf_dbg;      // phase timers of k_forest (diagnostic)
    uint32_t mrf_mask_words = 0;
    uint32_t mrf_tree_smem = 0, mrf_tree_cap = 0;
    b2::DevBuf<float> mrf_M;           // [3][nnz] messages child -> parent (k_tree)
    b2::DevBuf<uint16_t> mrf_J;        // [3][nnz] copy positions (k_tree)
    b2::DevBuf<uint4> mrf_rec;         // [3 F] 48-byte node records in forest order (k_tree_prep)
    b2::DevBuf<uint4> mrf_adj4;        // compact degree<=3 adjacency
    b2::DevBuf<uint32_t> mrf_queue;    // forest frontier lists + stamps
    b2::DevBuf<uint32_t> mrf_par;      // spanning-tree view selection only: parent of every node in the spanning forest
    b2::DevBuf<uint32_t> mrf_snap;     // spanning-tree view selection only: [2][F] labels and label positions at the start
                                       // of an iteration
    // the contracted MRF of multilevel view selection (mrf_multilevel.cu), grow-only scratch: node of every face, per node
    // label / label position / size / label-list offsets / CSR row / compact adjacency, coarse label lists and edges, and the
    // sort and scan buffers of the contraction (max(nnz, adjacency entries) each)
    b2::DevBuf<uint32_t> ml_region, ml_clabels, ml_clidx, ml_csize, ml_cadj_ptr, ml_cadj_idx, ml_cdeg, ml_changed;
    b2::DevBuf<uint64_t> ml_cptr, ml_cnt64;
    b2::DevBuf<uint4> ml_cadj4;
    b2::DevBuf<uint16_t> ml_cview;
    b2::DevBuf<float> ml_ccost, ml_cwgt;
    b2::DevBuf<uint32_t> ml_u32[3];
    b2::DevBuf<uint64_t> ml_key[2];
    b2::DevBuf<float> ml_f32;
    uint32_t ml_nodes = 0;
    uint32_t *mrf_host_flags = nullptr;   // pinned: stop flags the host polls behind the launches it queued
    unsigned long long mrf_forest_nodes = 0, mrf_forest_nnz = 0;   // summed over the iterations of the last run
    uint32_t mrf_slow_trees = 0;
    b2tex_mrf_params mrf_params{};
    int mrf_group = 32;

    // seam
    b2::DevBuf<uint32_t> vf_ptr, vf_idx, vv_ptr, vv_idx;
    // scratch of the mesh-graph build (graph.cu): sort keys [6F] x 2, values [3F] x 2, counts / run heads [6F], scalars
    b2::DevBuf<uint64_t> g_key[2];
    b2::DevBuf<uint32_t> g_val[2], g_cnt;
    b2::DevBuf<unsigned long long> g_scal;
    b2::DevBuf<uint32_t> row_ptr, row_label, arow_ptr, arow_rows;
    b2::DevBuf<float> arow_b;
    b2::DevBuf<uint32_t> csr_ptr, csr_col, csr_enc;
    b2::DevBuf<float> seam_dval;
    b2::DevBuf<float> csr_val, seam_diag, seam_rhs, seam_x, seam_r, seam_t;
    b2::DevBuf<float4> seam_p;
    b2::DevBuf<double> seam_partials;
    b2::DevBuf<uint32_t> seam_status;
    uint32_t R = 0, A_rows = 0;
    uint64_t nnz_L = 0;

    // texture patches (allocated on first use, released by patches_free)
    b2::PatchState *patches = nullptr;
    // peer-memory blocks of the multi-GPU seam solve (seam_mg.cu)
    b2::MgState *seam_mg = nullptr;
    // peer-memory block of the multi-GPU view selection (mrf.cu): c->labels lives inside it while it exists
    b2::MrfMgState *mrf_mg = nullptr;
};

namespace b2 {
// `bits` and everything derived from them are out of date
inline void invalidate(b2tex_ctx *c, uint32_t bits) { c->valid &= ~(bits | dependents_of(bits)); }
// `bits` were just (re)computed: everything derived from them is out of date, they are valid
inline void mark_valid(b2tex_ctx *c, uint32_t bits) { c->valid = (c->valid & ~dependents_of(bits)) | bits; }
// B2TEX_ERR_ARG naming the items of `bits` that are not valid
inline int require(b2tex_ctx *c, uint32_t bits, const char *stage)
{
    const uint32_t missing = bits & ~c->valid;
    if (!missing) return B2TEX_OK;
    std::string names;
    for (int i = 0; i < NUM_ITEMS; ++i)
        if (missing & (1u << i)) names += std::string(names.empty() ? "" : ", ") + item_name(i);
    set_error("%s: missing or out of date: %s", stage, names.c_str());
    return B2TEX_ERR_ARG;
}
// F faces without a mesh (view selection or data-cost postprocessing of caller arrays)
inline void set_face_count(b2tex_ctx *c, uint32_t F)
{
    invalidate(c, MESH);
    c->F = F; c->face_begin = 0; c->face_end = F;
}

// Records a pair of events around a launch sequence on the context's stream when profiling is on.
struct ScopedTimer {
    b2tex_ctx *c;
    size_t idx = (size_t)-1;
    ScopedTimer(b2tex_ctx *ctx, const char *name, double bytes = 0.0) : c(ctx)
    {
        if (!c->profile) return;
        KTimer t{name, nullptr, nullptr, bytes};
        if (cudaEventCreate(&t.a) != cudaSuccess || cudaEventCreate(&t.b) != cudaSuccess) return;
        cudaEventRecord(t.a, c->stream);
        idx = c->timers.size();
        c->timers.push_back(t);
    }
    ~ScopedTimer()
    {
        if (idx != (size_t)-1) cudaEventRecord(c->timers[idx].b, c->stream);
    }
};
// stage entry points implemented in the individual .cu files
int prepare_images(b2tex_ctx *c, int data_term, bool force = false);
int prepare_views(b2tex_ctx *c, int data_term);    // camera block only (no pixel data needed)
int wait_for_images(b2tex_ctx *c);                 // the compute stream waits for a deferred image upload
// flags[v] != 0: view v has a zero-sum corner pixel (it gets a validity mask); reads the camera block in views_dev
int zero_corner_flags(b2tex_ctx *c, std::vector<uint32_t> &flags);
int undistort_views(b2tex_ctx *c, const b2tex_distortion *d, uint32_t num_views);
int build_bvh(b2tex_ctx *c, bool force = false);
int data_costs_qualities(b2tex_ctx *c, const b2tex_settings *st, b2tex_dc_info *info);
int data_costs_histogram(b2tex_ctx *c, float gmax);
int data_costs_postprocess(b2tex_ctx *c, const b2tex_settings *st, uint32_t F, const uint64_t *face_ptr, const uint16_t *view,
                           const float *quality, const float *mean_ycbcr, b2tex_dc_info *info);
int data_costs_normalize(b2tex_ctx *c, float gmax, const uint32_t *bins_host, b2tex_dc_info *info);
int mrf_init(b2tex_ctx *c, const b2tex_mrf_params *p, int64_t *energy_fixed);
int mrf_iterate(b2tex_ctx *c, uint32_t t, int64_t *energy_fixed);
int mrf_run(b2tex_ctx *c, const b2tex_mrf_params *p, b2tex_mrf_info *info, double *trace);
int mrf_prepare(b2tex_ctx *c, const b2tex_mrf_params *p);
int mrf_energy_only(b2tex_ctx *c, int64_t *energy_fixed);
int mrf_sample_only(b2tex_ctx *c, const b2tex_mrf_params *p, uint32_t t, uint32_t *level_host);
int mrf_energy_double(b2tex_ctx *c, double *e, uint64_t *unseen);
// multilevel view selection (mrf_multilevel.cu): contract c->labels into the ml_* buffers; project the coarse labels
// back onto c->labels / c->mrf_lidx (a no-op once *stop != 0)
int mrf_contract(b2tex_ctx *c, uint32_t *num_nodes);
int mrf_project(b2tex_ctx *c, const uint32_t *stop);
int seam_run(b2tex_ctx *c, b2tex_seam_info *info, bool solve = true);
int seam_mg_export(b2tex_ctx *c, uint32_t rank, uint32_t nranks, void *handle64);
int seam_mg_import(b2tex_ctx *c, uint32_t peer_rank, const void *handle64);
int seam_mg_solve(b2tex_ctx *c, b2tex_seam_info *info);
void seam_mg_free(b2tex_ctx *c);
int mrf_mg_export(b2tex_ctx *c, uint32_t rank, uint32_t nranks, void *handle64);
int mrf_mg_import(b2tex_ctx *c, uint32_t peer_rank, const void *handle64);
void mrf_mg_free(b2tex_ctx *c);
int mrf_mg_attach(b2tex_ctx *c, uint32_t peer_rank, void *peer_block);
void *mrf_mg_block(b2tex_ctx *c);
int seam_mg_attach(b2tex_ctx *c, uint32_t peer_rank, void *peer_block);
void *seam_mg_block(b2tex_ctx *c);
int patches_run(b2tex_ctx *c, int apply_adjust, b2tex_patch_info *info);
int patches_download(b2tex_ctx *c, int32_t *desc, uint32_t *faces, float *texcoords, float *images, uint8_t *validity,
                     uint8_t *blending);
void patches_free(b2tex_ctx *c);
int local_seam_run(b2tex_ctx *c, b2tex_local_seam_info *info);
int build_mesh_graph(b2tex_ctx *c, b2tex_graph_info *info);
// k_graph_validate: B2TEX_ERR_ARG naming the lowest face with an index >= nv ("<fn>: face ..."); sets up c->g_scal
int validate_faces(b2tex_ctx *c, const uint32_t *faces, uint32_t F, uint32_t nv, const char *fn, const char *timer);
// tex::prepare_mesh on the raw mesh resident in verts / faces (F, Vn set, MESH not valid)
int prepare_mesh(b2tex_ctx *c, b2tex_mesh_prep_info *info);
int cub_exclusive_sum_u64(b2tex_ctx *c, const uint64_t *in, uint64_t *out, size_t n);
int cub_exclusive_sum_u32(b2tex_ctx *c, const uint32_t *in, uint32_t *out, size_t n);
}  // namespace b2
