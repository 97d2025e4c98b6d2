// api.cu -- extern "C" entry points declared in include/b2tex.h.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

#include <atomic>
#include <mutex>

namespace b2 {
static std::atomic<unsigned long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
static thread_local char g_err[1024] = "";
void set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
}  // namespace b2

using namespace b2;

extern "C" {

const char *b2tex_last_error(void) { return g_err; }
void b2tex_free(void *p) { free(p); }

void b2tex_default_mrf_params(b2tex_mrf_params *p)
{
    p->max_iterations = 100;
    p->rounds = 16;     // forest growth rounds: same coverage (0.695 of the nodes) as 32 / 256 with half the
    p->root_div = 64;   // grid-wide barriers; energies within 0.5 % (DESIGN.md, solver table)
    p->seed = 548923723u;  // view_selection.cpp:115
    p->window = 5;         // view_selection.cpp:84
    p->ratio = 0.01f;
    p->num_parts = 1;
    p->num_views = 0;
    p->use_multilevel = 0;
    p->use_spanning_tree = 0;
    p->spanning_tree_multilevel_after_n_iterations = 0;
}

void b2tex_texrecon_mrf_params(b2tex_mrf_params *p)
{
    b2tex_default_mrf_params(p);
    p->use_spanning_tree = 1;
    p->use_multilevel = 1;
    p->spanning_tree_multilevel_after_n_iterations = 5;   // view_selection.cpp:103-115
}

int b2tex_create(int device, b2tex_ctx **out)
{
    if (!out) { set_error("b2tex_create: out is null"); return B2TEX_ERR_ARG; }
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        set_error("no CUDA device available (%s); this library has no CPU fallback",
                  e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
        return B2TEX_ERR_CUDA;
    }
    if (device < 0 || device >= ndev) { set_error("device %d out of range (%d)", device, ndev); return B2TEX_ERR_ARG; }
    B2_CUDA(cudaSetDevice(device));
    b2tex_ctx *c = new b2tex_ctx();
    c->device = device;
    cudaDeviceProp prop;
    B2_CUDA(cudaGetDeviceProperties(&prop, device));
    c->num_sms = prop.multiProcessorCount;
    B2_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    B2_CUDA(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    B2_CUDA(cudaEventCreateWithFlags(&c->images_uploaded, cudaEventDisableTiming));
    *out = c;
    return B2TEX_OK;
}

void b2tex_destroy(b2tex_ctx *c)
{
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    patches_free(c);
    seam_mg_free(c);
    mrf_mg_free(c);
    if (c->mrf_host_flags) cudaFreeHost(c->mrf_host_flags);
    if (c->images_uploaded) cudaEventDestroy(c->images_uploaded);
    if (c->copy_stream) { cudaStreamSynchronize(c->copy_stream); cudaStreamDestroy(c->copy_stream); }
    cudaStreamDestroy(c->stream);
    delete c;
}

uint64_t b2tex_launch_count(void) { return (uint64_t)b2::g_launches.load(); }
uint64_t b2tex_stream(b2tex_ctx *c) { return (uint64_t)(uintptr_t)c->stream; }

int b2tex_profile(b2tex_ctx *c, int enable)
{
    B2_CUDA(cudaSetDevice(c->device));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    for (auto &t : c->timers) { cudaEventDestroy(t.a); cudaEventDestroy(t.b); }
    c->timers.clear();
    c->profile = enable != 0;
    return B2TEX_OK;
}

// "name ms bytes" per recorded launch group, newline separated; returns the number of records
int b2tex_profile_report(b2tex_ctx *c, char *buf, uint64_t cap)
{
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    size_t off = 0;
    int n = 0;
    if (cap) buf[0] = 0;
    for (auto &t : c->timers) {
        float ms = 0.0f;
        if (cudaEventElapsedTime(&ms, t.a, t.b) != cudaSuccess) continue;
        int w = snprintf(buf + off, off < cap ? cap - off : 0, "%s %.6f %.0f\n", t.name, ms, t.bytes);
        if (w < 0 || off + (size_t)w >= cap) break;
        off += (size_t)w;
        ++n;
    }
    return n;
}

int b2tex_device_synchronize(b2tex_ctx *c)
{
    B2_CUDA(cudaSetDevice(c->device));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    return B2TEX_OK;
}

}  // extern "C"

// Uploads the vertices, the faces and (when given) the face normals and forgets everything derived from an earlier mesh.
// The mesh is not marked valid: the caller does that.
static int upload_mesh(b2tex_ctx *c, const float *verts, uint32_t nv, const uint32_t *faces, const float *normals,
                       uint32_t nf)
{
    invalidate(c, MESH);
    c->Vn = nv; c->F = nf; c->face_begin = 0; c->face_end = nf;
    B2_TRY(c->verts.upload(verts, 3 * (size_t)nv, c->stream));
    B2_TRY(c->faces.upload(faces, 3 * (size_t)nf, c->stream));
    if (normals) B2_TRY(c->normals.upload(normals, 3 * (size_t)nf, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    return B2TEX_OK;
}

extern "C" {

int b2tex_set_mesh(b2tex_ctx *c, const float *verts, uint32_t nv, const uint32_t *faces, const float *normals,
                   uint32_t nf)
{
    B2_CUDA(cudaSetDevice(c->device));
    if (!verts || !faces || !normals) { set_error("set_mesh: null pointer"); return B2TEX_ERR_ARG; }
    B2_TRY(upload_mesh(c, verts, nv, faces, normals, nf));
    mark_valid(c, MESH);
    return B2TEX_OK;
}

int b2tex_prepare_mesh(b2tex_ctx *c, const float *verts, uint32_t nv, const uint32_t *faces, uint32_t nf,
                       b2tex_mesh_prep_info *info)
{
    B2_CUDA(cudaSetDevice(c->device));
    invalidate(c, MESH);
    if (!verts || !faces) { set_error("prepare_mesh: null pointer"); return B2TEX_ERR_ARG; }
    if (nf == 0) { set_error("prepare_mesh: the mesh has no faces"); return B2TEX_ERR_ARG; }
    int rc = upload_mesh(c, verts, nv, faces, nullptr, nf);
    if (rc == B2TEX_OK) rc = prepare_mesh(c, info);
    if (rc != B2TEX_OK) invalidate(c, MESH);   // no mesh, graph or prepared arrays survive a failure
    return rc;
}

int b2tex_prepared_mesh_download(b2tex_ctx *c, uint32_t *faces, float *face_normals, float *vertex_normals,
                                 uint32_t *kept_face_ids)
{
    B2_CUDA(cudaSetDevice(c->device));
    B2_TRY(require(c, PREP, "prepared_mesh_download"));
    if (faces) B2_TRY(c->faces.download(faces, 3 * (size_t)c->F, c->stream));
    if (face_normals) B2_TRY(c->normals.download(face_normals, 3 * (size_t)c->F, c->stream));
    if (vertex_normals) B2_TRY(c->vnormals.download(vertex_normals, 3 * (size_t)c->Vn, c->stream));
    if (kept_face_ids) B2_TRY(c->kept_ids.download(kept_face_ids, c->F, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    return B2TEX_OK;
}

int b2tex_set_face_range(b2tex_ctx *c, uint32_t fb, uint32_t fe)
{
    if (fb > fe || fe > c->F) { set_error("bad face range"); return B2TEX_ERR_ARG; }
    c->face_begin = fb; c->face_end = fe;
    invalidate(c, COSTS);
    return B2TEX_OK;
}

int b2tex_set_views(b2tex_ctx *c, const b2tex_view *views, uint32_t K)
{
    B2_CUDA(cudaSetDevice(c->device));
    if (K > 65535u) { set_error("Exeeded maximal number of views"); return B2TEX_ERR_LIMITS; }
    invalidate(c, VIEWS);
    c->K = K;
    c->views_host.assign(views, views + K);
    c->img_off.assign((size_t)K + 1, 0);
    for (uint32_t v = 0; v < K; ++v) {
        if (views[v].width < 2 || views[v].height < 2 || !views[v].rgb) { set_error("view %u: bad image", v); return B2TEX_ERR_ARG; }
        c->img_off[v + 1] = c->img_off[v] + (size_t)views[v].width * views[v].height;
    }
    // a view with a zero-sum corner pixel gets a validity mask (texture_view.cpp:42-94), which the cull already reads
    // (TextureView::inside -> valid_pixel): such scenes need their pixels first.  Four pixels per view, read on the host.
    c->any_corner_flag = false;
    for (uint32_t v = 0; v < K; ++v) {
        const uint8_t *img = (const uint8_t *)views[v].rgb;
        const size_t w = (size_t)views[v].width, h = (size_t)views[v].height;
        const size_t corner[4] = {0, w - 1, (h - 1) * w, (h - 1) * w + w - 1};
        for (size_t o : corner)
            if ((int)img[3 * o] + img[3 * o + 1] + img[3 * o + 2] == 0) c->any_corner_flag = true;
    }
    B2_TRY(c->rgb.alloc(3 * c->img_off[K]));
    // deferred (one-shot entry points only: the caller's buffers stay valid until the call returns): the copies go to the
    // copy stream and the stage that first touches pixels waits for them (wait_for_images); otherwise: done on return
    cudaStream_t cs = c->defer_image_sync ? c->copy_stream : c->stream;
    if (c->defer_image_sync) B2_CUDA(cudaStreamSynchronize(c->stream));   // the previous use of the image buffer is over
    for (uint32_t v = 0; v < K; ++v) {
        size_t px = (size_t)views[v].width * views[v].height;
        B2_CUDA(cudaMemcpyAsync(c->rgb.p + 3 * c->img_off[v], views[v].rgb, 3 * px, cudaMemcpyHostToDevice, cs));
        c->views_host[v].rgb = nullptr;
    }
    if (c->defer_image_sync) {
        B2_CUDA(cudaEventRecord(c->images_uploaded, cs));
        c->images_in_flight = true;
    } else {
        B2_CUDA(cudaStreamSynchronize(c->stream));
        c->images_in_flight = false;
    }
    mark_valid(c, VIEWS | PIXELS);
    return B2TEX_OK;
}

int b2tex_undistort_views(b2tex_ctx *c, const b2tex_distortion *d, uint32_t num_views)
{
    B2_CUDA(cudaSetDevice(c->device));
    return undistort_views(c, d, num_views);
}

int b2tex_set_adjacency(b2tex_ctx *c, const uint32_t *adj_ptr, const uint32_t *adj_idx)
{
    B2_CUDA(cudaSetDevice(c->device));
    if (!c->F) { set_error("set_adjacency: set the mesh (or data costs) first"); return B2TEX_ERR_ARG; }
    invalidate(c, ADJ);
    B2_TRY(c->adj_ptr.upload(adj_ptr, (size_t)c->F + 1, c->stream));
    B2_TRY(c->adj_idx.upload(adj_idx, adj_ptr[c->F], c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    mark_valid(c, ADJ);
    return B2TEX_OK;
}

int b2tex_set_vertex_rings(b2tex_ctx *c, const uint32_t *vf_ptr, const uint32_t *vf_idx, const uint32_t *vv_ptr,
                           const uint32_t *vv_idx)
{
    B2_CUDA(cudaSetDevice(c->device));
    if (!c->Vn) { set_error("set_vertex_rings: set the mesh first"); return B2TEX_ERR_ARG; }
    invalidate(c, RINGS);
    B2_TRY(c->vf_ptr.upload(vf_ptr, (size_t)c->Vn + 1, c->stream));
    B2_TRY(c->vf_idx.upload(vf_idx, vf_ptr[c->Vn], c->stream));
    B2_TRY(c->vv_ptr.upload(vv_ptr, (size_t)c->Vn + 1, c->stream));
    B2_TRY(c->vv_idx.upload(vv_idx, vv_ptr[c->Vn], c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    mark_valid(c, RINGS);
    return B2TEX_OK;
}

int b2tex_build_mesh_graph(b2tex_ctx *c, b2tex_graph_info *info)
{
    B2_CUDA(cudaSetDevice(c->device));
    return build_mesh_graph(c, info);
}

int b2tex_mesh_graph_download(b2tex_ctx *c, uint32_t *adj_ptr, uint32_t *adj_idx, uint32_t *vf_ptr, uint32_t *vf_idx,
                              uint32_t *vv_ptr, uint32_t *vv_idx)
{
    B2_CUDA(cudaSetDevice(c->device));
    if (!(c->valid & (ADJ | RINGS))) { set_error("mesh_graph_download: no graph is resident"); return B2TEX_ERR_ARG; }
    if (adj_ptr || adj_idx) B2_TRY(require(c, ADJ, "mesh_graph_download"));
    if (vf_ptr || vf_idx || vv_ptr || vv_idx) B2_TRY(require(c, RINGS, "mesh_graph_download"));
    if (adj_ptr) B2_TRY(c->adj_ptr.download(adj_ptr, (size_t)c->F + 1, c->stream));
    if (adj_idx) B2_TRY(c->adj_idx.download(adj_idx, c->adj_idx.n, c->stream));
    if (vf_ptr) B2_TRY(c->vf_ptr.download(vf_ptr, (size_t)c->Vn + 1, c->stream));
    if (vf_idx) B2_TRY(c->vf_idx.download(vf_idx, c->vf_idx.n, c->stream));
    if (vv_ptr) B2_TRY(c->vv_ptr.download(vv_ptr, (size_t)c->Vn + 1, c->stream));
    if (vv_idx) B2_TRY(c->vv_idx.download(vv_idx, c->vv_idx.n, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    return B2TEX_OK;
}

int b2tex_set_data_costs(b2tex_ctx *c, const uint64_t *face_ptr, const uint16_t *view, const float *cost)
{
    B2_CUDA(cudaSetDevice(c->device));
    if (!c->F) { set_error("set_data_costs: number of faces unknown (set mesh first)"); return B2TEX_ERR_ARG; }
    uint64_t nnz = face_ptr[c->F];
    invalidate(c, COSTS);
    B2_TRY(c->dc_ptr.upload(face_ptr, (size_t)c->F + 1, c->stream));
    B2_TRY(c->dc_view.upload(view, nnz, c->stream));
    B2_TRY(c->dc_cost.upload(cost, nnz, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    c->nnz = nnz;
    mark_valid(c, COSTS);
    return B2TEX_OK;
}

int b2tex_set_labels(b2tex_ctx *c, const uint32_t *labels)
{
    B2_CUDA(cudaSetDevice(c->device));
    if (c->K)   // texrecon.cpp:141-153 rejects such labelings ("Incorrect labeling"); the seam / patch kernels index views[label - 1]
        for (uint32_t i = 0; i < c->F; ++i)
            if (labels[i] > c->K) { set_error("Incorrect labeling (face %u has label %u, %u views)", i, labels[i], c->K); return B2TEX_ERR_LABELING; }
    invalidate(c, LABELS);
    B2_TRY(c->labels.upload(labels, c->F, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    mark_valid(c, LABELS);
    return B2TEX_OK;
}

int b2tex_data_costs_qualities(b2tex_ctx *c, const b2tex_settings *st, b2tex_dc_info *info)
{
    B2_CUDA(cudaSetDevice(c->device));
    return data_costs_qualities(c, st, info);
}

int b2tex_data_costs_histogram(b2tex_ctx *c, float gmax, uint32_t *bins, int to_host)
{
    B2_CUDA(cudaSetDevice(c->device));
    B2_TRY(data_costs_histogram(c, gmax));
    if (bins && to_host) {
        B2_TRY(c->hist.download(bins, 10000, c->stream));
        B2_CUDA(cudaStreamSynchronize(c->stream));
    }
    return B2TEX_OK;
}

int b2tex_data_costs_normalize(b2tex_ctx *c, float gmax, const uint32_t *bins, b2tex_dc_info *info)
{
    B2_CUDA(cudaSetDevice(c->device));
    return data_costs_normalize(c, gmax, bins, info);
}

int b2tex_data_costs_run(b2tex_ctx *c, const b2tex_settings *st, b2tex_dc_info *info)
{
    B2_CUDA(cudaSetDevice(c->device));
    B2_TRY(data_costs_qualities(c, st, info));
    float gmax = info->max_quality;
    uint32_t *bins = (uint32_t *)malloc(10000 * sizeof(uint32_t));
    int rc = b2tex_data_costs_histogram(c, gmax, bins, 1);
    if (rc == B2TEX_OK) {
        uint64_t cand = info->candidates, rays = info->rays;
        rc = data_costs_normalize(c, gmax, bins, info);
        info->candidates = cand; info->rays = rays;
    }
    free(bins);
    return rc;
}

int b2tex_data_costs_download(b2tex_ctx *c, uint64_t *face_ptr, uint16_t *view, float *cost, float *quality)
{
    B2_CUDA(cudaSetDevice(c->device));
    B2_TRY(require(c, COSTS, "data_costs_download"));
    if (face_ptr) B2_TRY(c->dc_ptr.download(face_ptr, (size_t)c->F + 1, c->stream));
    if (view) B2_TRY(c->dc_view.download(view, c->nnz, c->stream));
    if (cost) B2_TRY(c->dc_cost.download(cost, c->nnz, c->stream));
    if (quality) B2_TRY(c->dc_quality.download(quality, c->nnz, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    return B2TEX_OK;
}

int b2tex_mrf_init(b2tex_ctx *c, const b2tex_mrf_params *p, int64_t *efix)
{
    B2_CUDA(cudaSetDevice(c->device));
    return mrf_init(c, p, efix);
}
int b2tex_mrf_iterate(b2tex_ctx *c, uint32_t t, int64_t *efix)
{
    B2_CUDA(cudaSetDevice(c->device));
    return mrf_iterate(c, t, efix);
}
int b2tex_mrf_energy(b2tex_ctx *c, int64_t *efix)
{
    B2_CUDA(cudaSetDevice(c->device));
    return mrf_energy_only(c, efix);
}
int b2tex_mrf_sample_forest(b2tex_ctx *c, const b2tex_mrf_params *p, uint32_t t, uint32_t *level)
{
    B2_CUDA(cudaSetDevice(c->device));
    return mrf_sample_only(c, p, t, level);
}

int b2tex_mrf_mg_export(b2tex_ctx *c, uint32_t rank, uint32_t num_ranks, void *ipc_handle_64_bytes)
{
    B2_CUDA(cudaSetDevice(c->device));
    return mrf_mg_export(c, rank, num_ranks, ipc_handle_64_bytes);
}
int b2tex_mrf_mg_import(b2tex_ctx *c, uint32_t peer_rank, const void *ipc_handle_64_bytes)
{
    B2_CUDA(cudaSetDevice(c->device));
    return mrf_mg_import(c, peer_rank, ipc_handle_64_bytes);
}

uint64_t b2tex_peer_block(b2tex_ctx *c, int which)
{
    return (uint64_t)(uintptr_t)(which == 0 ? mrf_mg_block(c) : seam_mg_block(c));
}
int b2tex_peer_attach(b2tex_ctx *c, int which, uint32_t peer_rank, uint64_t peer_block_device_ptr)
{
    B2_CUDA(cudaSetDevice(c->device));
    void *p = (void *)(uintptr_t)peer_block_device_ptr;
    return which == 0 ? mrf_mg_attach(c, peer_rank, p) : seam_mg_attach(c, peer_rank, p);
}

int b2tex_view_selection_prepare(b2tex_ctx *c, const b2tex_mrf_params *params)
{
    B2_CUDA(cudaSetDevice(c->device));
    b2tex_mrf_params p;
    if (params) p = *params; else b2tex_default_mrf_params(&p);
    B2_TRY(mrf_prepare(c, &p));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    return B2TEX_OK;
}

int b2tex_view_selection_run(b2tex_ctx *c, const b2tex_mrf_params *params, b2tex_mrf_info *info, double *trace)
{
    B2_CUDA(cudaSetDevice(c->device));
    b2tex_mrf_params p;
    if (params) p = *params; else b2tex_default_mrf_params(&p);
    if (p.window == 0) p.window = 1;
    if (p.max_iterations + 2 > 1024u) { set_error("view selection: at most 1022 iterations"); return B2TEX_ERR_ARG; }
    return mrf_run(c, &p, info, trace);
}

int b2tex_labels_download(b2tex_ctx *c, uint32_t *labels)
{
    B2_CUDA(cudaSetDevice(c->device));
    B2_TRY(require(c, LABELS, "labels_download"));
    B2_TRY(c->labels.download(labels, c->F, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    return B2TEX_OK;
}

int b2tex_texture_patches_run(b2tex_ctx *c, int apply_adjust, b2tex_patch_info *info)
{
    B2_CUDA(cudaSetDevice(c->device));
    b2tex_patch_info local;
    return patches_run(c, apply_adjust, info ? info : &local);
}

int b2tex_local_seam_leveling_run(b2tex_ctx *c, b2tex_local_seam_info *info)
{
    B2_CUDA(cudaSetDevice(c->device));
    b2tex_local_seam_info local;
    return local_seam_run(c, info ? info : &local);
}

int b2tex_texture_patches_download(b2tex_ctx *c, int32_t *desc, uint32_t *faces, float *texcoords, float *images,
                                   uint8_t *validity, uint8_t *blending)
{
    B2_CUDA(cudaSetDevice(c->device));
    return patches_download(c, desc, faces, texcoords, images, validity, blending);
}

int b2tex_seam_run(b2tex_ctx *c, b2tex_seam_info *info)
{
    B2_CUDA(cudaSetDevice(c->device));
    return seam_run(c, info);
}

// ---- multi-GPU seam solve: assembly on every rank, then one fused compute + exchange kernel per GPU (seam_mg.cu) ----
int b2tex_seam_assemble(b2tex_ctx *c, b2tex_seam_info *info)
{
    B2_CUDA(cudaSetDevice(c->device));
    return seam_run(c, info, false);
}

int b2tex_seam_mg_export(b2tex_ctx *c, uint32_t rank, uint32_t num_ranks, void *ipc_handle_64_bytes)
{
    B2_CUDA(cudaSetDevice(c->device));
    return seam_mg_export(c, rank, num_ranks, ipc_handle_64_bytes);
}

int b2tex_seam_mg_import(b2tex_ctx *c, uint32_t peer_rank, const void *ipc_handle_64_bytes)
{
    B2_CUDA(cudaSetDevice(c->device));
    return seam_mg_import(c, peer_rank, ipc_handle_64_bytes);
}

int b2tex_seam_mg_solve(b2tex_ctx *c, b2tex_seam_info *info)
{
    B2_CUDA(cudaSetDevice(c->device));
    return seam_mg_solve(c, info);
}

int b2tex_seam_download(b2tex_ctx *c, uint32_t *row_ptr, uint32_t *row_label, float *x, float *rhs)
{
    B2_CUDA(cudaSetDevice(c->device));
    B2_TRY(require(c, SEAM, "seam_download"));
    const size_t R = c->R;
    if (row_ptr) B2_TRY(c->row_ptr.download(row_ptr, (size_t)c->Vn + 1, c->stream));
    if (row_label) B2_TRY(c->row_label.download(row_label, R, c->stream));
    std::vector<float> tmp(3 * R);
    for (int pass = 0; pass < 2; ++pass) {
        float *dst = pass == 0 ? x : rhs;
        if (!dst) continue;
        B2_TRY((pass == 0 ? c->seam_x : c->seam_rhs).download(tmp.data(), 3 * R, c->stream));
        B2_CUDA(cudaStreamSynchronize(c->stream));
        for (size_t r = 0; r < R; ++r)
            for (int ch = 0; ch < 3; ++ch) dst[3 * r + ch] = tmp[(size_t)ch * R + r];
    }
    B2_CUDA(cudaStreamSynchronize(c->stream));
    return B2TEX_OK;
}

int b2tex_seam_matrix_download(b2tex_ctx *c, uint32_t *csr_ptr, uint32_t *csr_col, float *csr_val)
{
    B2_CUDA(cudaSetDevice(c->device));
    B2_TRY(require(c, SEAM, "seam_matrix_download"));
    B2_TRY(c->csr_ptr.download(csr_ptr, (size_t)c->R + 1, c->stream));
    B2_TRY(c->csr_col.download(csr_col, c->nnz_L, c->stream));
    B2_TRY(c->csr_val.download(csr_val, c->nnz_L, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    return B2TEX_OK;
}

uint64_t b2tex_device_ptr(b2tex_ctx *c, const char *name, uint64_t *n)
{
    uint64_t p = 0, cnt = 0;
#define B2_NAME(nm, buf) if (!strcmp(name, nm)) { p = (uint64_t)(uintptr_t)(buf).p; cnt = (buf).n; }
    B2_NAME("labels", c->labels)
    B2_NAME("dc_ptr", c->dc_ptr)
    B2_NAME("dc_view", c->dc_view)
    B2_NAME("dc_cost", c->dc_cost)
    B2_NAME("dc_quality", c->dc_quality)
    B2_NAME("hist", c->hist)
    B2_NAME("seam_x", c->seam_x)
    B2_NAME("rgb", c->rgb)
    B2_NAME("grad", c->grad)
#undef B2_NAME
    if (n) *n = cnt;
    return p;
}

// ---- one-shot host-buffer entry points ---------------------------------------------------------
// A one-shot call needs a context: a stream plus some sixty device buffers (3 GB at C3).  Creating and destroying them
// per call costs more than the kernels (cudaMalloc / cudaFree serialise the device), so finished one-shot calls park
// their context here (buffers are grow-only and every stage re-derives its state from the set_* calls) and the next
// call on the same device picks it up.  b2tex_release_cached_contexts() frees them.
static std::mutex g_pool_mu;
static std::vector<b2tex_ctx *> g_pool;
constexpr size_t POOL_MAX = 2;

static int acquire_ctx(b2tex_ctx **out)
{
    int device = 0;
    if (cudaGetDevice(&device) != cudaSuccess) device = 0;   // the calling thread's current device, like any runtime-API call
    {
        std::lock_guard<std::mutex> lk(g_pool_mu);
        for (size_t i = 0; i < g_pool.size(); ++i)
            if (g_pool[i]->device == device) {
                b2tex_ctx *c = g_pool[i];
                g_pool.erase(g_pool.begin() + (long)i);
                invalidate(c, ALL_ITEMS);
                c->Vn = c->F = c->K = 0; c->face_begin = c->face_end = 0; c->nnz = 0; c->R = 0;
                *out = c;
                return B2TEX_OK;
            }
    }
    return b2tex_create(device, out);
}

static void release_ctx(b2tex_ctx *c, int rc)
{
    if (!c) return;
    if (rc == B2TEX_OK && cudaStreamSynchronize(c->stream) == cudaSuccess && !c->profile) {
        std::lock_guard<std::mutex> lk(g_pool_mu);
        if (g_pool.size() < POOL_MAX) { g_pool.push_back(c); return; }
    }
    b2tex_destroy(c);   // failed calls never hand their context on
}

void b2tex_release_cached_contexts(void)
{
    std::vector<b2tex_ctx *> v;
    { std::lock_guard<std::mutex> lk(g_pool_mu); v.swap(g_pool); }
    for (b2tex_ctx *c : v) b2tex_destroy(c);
}

// topology arrays of a one-shot call: 0 = all given, 1 = all NULL (derived on the device), -1 = a mix (error set)
static int topology_nulls(const char *fn, std::initializer_list<const uint32_t *> arrays)
{
    size_t nulls = 0;
    for (const uint32_t *a : arrays) nulls += a == nullptr;
    if (nulls == 0) return 0;
    if (nulls == arrays.size()) return 1;
    set_error("%s: the topology arrays must be all given or all NULL (%zu of %zu are NULL)", fn, nulls, arrays.size());
    return -1;
}

static int dc_oneshot(const float *verts, uint32_t nv, const uint32_t *faces, const float *normals, uint32_t nf,
                      const b2tex_view *views, uint32_t K, const b2tex_settings *st, b2tex_dc_info *info,
                      b2tex_ctx **out)
{
    if (K > 65535u) { set_error("Exeeded maximal number of views"); return B2TEX_ERR_LIMITS; }
    b2tex_ctx *c = nullptr;
    B2_TRY(acquire_ctx(&c));
    int rc = b2tex_set_mesh(c, verts, nv, faces, normals, nf);
    if (rc == B2TEX_OK) rc = b2tex_set_views(c, views, K);
    if (rc == B2TEX_OK) rc = b2tex_data_costs_run(c, st, info);
    if (rc != B2TEX_OK) { release_ctx(c, rc); return rc; }
    *out = c;
    return B2TEX_OK;
}

int b2tex_calculate_data_costs(const float *verts, uint32_t nv, const uint32_t *faces, const float *normals,
                               uint32_t nf, const b2tex_view *views, uint32_t K, const b2tex_settings *st,
                               uint64_t **face_ptr_out, uint16_t **view_out, float **cost_out, b2tex_dc_info *info)
{
    b2tex_ctx *c = nullptr;
    B2_TRY(dc_oneshot(verts, nv, faces, normals, nf, views, K, st, info, &c));
    *face_ptr_out = (uint64_t *)malloc(sizeof(uint64_t) * ((size_t)nf + 1));
    *view_out = (uint16_t *)malloc(sizeof(uint16_t) * (info->nnz ? info->nnz : 1));
    *cost_out = (float *)malloc(sizeof(float) * (info->nnz ? info->nnz : 1));
    int rc = b2tex_data_costs_download(c, *face_ptr_out, *view_out, *cost_out, nullptr);
    release_ctx(c, rc);
    return rc;
}

int b2tex_calculate_data_costs_into(const float *verts, uint32_t nv, const uint32_t *faces, const float *normals,
                                    uint32_t nf, const b2tex_view *views, uint32_t K, const b2tex_settings *st,
                                    uint64_t *face_ptr, uint16_t *view, float *cost, uint64_t capacity,
                                    b2tex_dc_info *info)
{
    b2tex_ctx *c = nullptr;
    B2_TRY(dc_oneshot(verts, nv, faces, normals, nf, views, K, st, info, &c));
    int rc = B2TEX_OK;
    if (info->nnz > capacity) {
        set_error("data costs need %llu entries, caller provided %llu", (unsigned long long)info->nnz,
                  (unsigned long long)capacity);
        rc = B2TEX_ERR_ARG;
    } else {
        rc = b2tex_data_costs_download(c, face_ptr, view, cost, nullptr);
    }
    release_ctx(c, rc);
    return rc;
}

int b2tex_postprocess_face_infos(uint32_t nf, const uint64_t *face_ptr, const uint16_t *view, const float *quality,
                                 const float *mean_color_ycbcr, const b2tex_settings *st, uint64_t *face_ptr_out,
                                 uint16_t *view_out, float *cost_out, b2tex_dc_info *info)
{
    b2tex_ctx *c = nullptr;
    B2_TRY(acquire_ctx(&c));
    b2tex_dc_info local;
    if (!info) info = &local;
    int rc = data_costs_postprocess(c, st, nf, face_ptr, view, quality, mean_color_ycbcr, info);
    if (rc == B2TEX_OK) {
        const float gmax = info->max_quality;
        uint32_t *bins = (uint32_t *)malloc(10000 * sizeof(uint32_t));
        rc = b2tex_data_costs_histogram(c, gmax, bins, 1);
        if (rc == B2TEX_OK) {
            const uint64_t cand = info->candidates;
            rc = data_costs_normalize(c, gmax, bins, info);
            info->candidates = cand; info->rays = 0;
        }
        free(bins);
    }
    if (rc == B2TEX_OK) rc = b2tex_data_costs_download(c, face_ptr_out, view_out, cost_out, nullptr);
    release_ctx(c, rc);
    return rc;
}

int b2tex_view_selection(uint32_t nf, const uint32_t *adj_ptr, const uint32_t *adj_idx, const uint64_t *face_ptr,
                         const uint16_t *view, const float *cost, const b2tex_mrf_params *params,
                         uint32_t *labels_out, b2tex_mrf_info *info)
{
    b2tex_ctx *c = nullptr;
    B2_TRY(acquire_ctx(&c));
    set_face_count(c, nf);
    // DataCosts::rows() (= number of views) is not part of the CSR: params->num_views if the caller
    // knows it, otherwise bounded from the content (one host pass over nnz)
    uint32_t K = params ? params->num_views : 0;
    if (K == 0) {
        uint32_t maxview = 0;
        for (uint64_t i = 0; i < face_ptr[nf]; ++i) maxview = view[i] > maxview ? view[i] : maxview;
        K = face_ptr[nf] ? maxview + 1 : 0;
    }
    c->K = K;
    int rc = b2tex_set_data_costs(c, face_ptr, view, cost);
    if (rc == B2TEX_OK) rc = b2tex_set_adjacency(c, adj_ptr, adj_idx);
    if (rc == B2TEX_OK) rc = b2tex_view_selection_run(c, params, info, nullptr);
    if (rc == B2TEX_OK) rc = b2tex_labels_download(c, labels_out);
    release_ctx(c, rc);
    return rc;
}

int b2tex_global_seam_leveling(const float *verts, uint32_t nv, const uint32_t *faces, uint32_t nf,
                               const uint32_t *vf_ptr, const uint32_t *vf_idx, const uint32_t *vv_ptr,
                               const uint32_t *vv_idx, const uint32_t *labels, const b2tex_view *views, uint32_t K,
                               uint32_t *row_ptr_out, uint32_t **row_label_out, float **x_out, b2tex_seam_info *info)
{
    const int derive = topology_nulls("global_seam_leveling", {vf_ptr, vf_idx, vv_ptr, vv_idx});
    if (derive < 0) return B2TEX_ERR_ARG;
    b2tex_ctx *c = nullptr;
    B2_TRY(acquire_ctx(&c));
    std::vector<float> dummy_normals(3 * (size_t)nf, 0.0f);
    int rc = b2tex_set_mesh(c, verts, nv, faces, dummy_normals.data(), nf);
    if (rc == B2TEX_OK) rc = b2tex_set_views(c, views, K);
    if (rc == B2TEX_OK) rc = derive ? b2tex_build_mesh_graph(c, nullptr) : b2tex_set_vertex_rings(c, vf_ptr, vf_idx, vv_ptr, vv_idx);
    if (rc == B2TEX_OK) rc = b2tex_set_labels(c, labels);
    if (rc == B2TEX_OK) rc = b2tex_seam_run(c, info);
    if (rc == B2TEX_OK) {
        *row_label_out = (uint32_t *)malloc(sizeof(uint32_t) * (info->num_rows ? info->num_rows : 1));
        *x_out = (float *)malloc(sizeof(float) * 3 * (info->num_rows ? info->num_rows : 1));
        rc = b2tex_seam_download(c, row_ptr_out, *row_label_out, *x_out, nullptr);
    }
    release_ctx(c, rc);
    return rc;
}

int b2tex_seam_leveling_patches(const float *verts, uint32_t nv, const uint32_t *faces, uint32_t nf, const uint32_t *adj_ptr,
                                const uint32_t *adj_idx, const uint32_t *vf_ptr, const uint32_t *vf_idx, const uint32_t *vv_ptr,
                                const uint32_t *vv_idx, const uint32_t *labels, const b2tex_view *views, uint32_t K, int do_global,
                                int do_local, int32_t **desc_out, uint32_t **faces_out, float **texcoords_out, float **images_out,
                                uint8_t **validity_out, b2tex_patch_info *pi, b2tex_seam_info *si, b2tex_local_seam_info *li)
{
    if (K > 65535u) { set_error("Exeeded maximal number of views"); return B2TEX_ERR_LIMITS; }
    const int derive = topology_nulls("seam_leveling_patches", {adj_ptr, adj_idx, vf_ptr, vf_idx, vv_ptr, vv_idx});
    if (derive < 0) return B2TEX_ERR_ARG;
    b2tex_ctx *c = nullptr;
    B2_TRY(acquire_ctx(&c));
    b2tex_patch_info pl; b2tex_seam_info sl; b2tex_local_seam_info ll;
    if (!pi) pi = &pl;
    if (!si) si = &sl;
    if (!li) li = &ll;
    memset(si, 0, sizeof(*si)); memset(li, 0, sizeof(*li));
    std::vector<float> dummy_normals(3 * (size_t)nf, 0.0f);
    int rc = b2tex_set_mesh(c, verts, nv, faces, dummy_normals.data(), nf);
    if (rc == B2TEX_OK) rc = b2tex_set_views(c, views, K);
    if (rc == B2TEX_OK && derive) rc = b2tex_build_mesh_graph(c, nullptr);
    if (rc == B2TEX_OK && !derive) rc = b2tex_set_adjacency(c, adj_ptr, adj_idx);
    if (rc == B2TEX_OK && !derive) rc = b2tex_set_vertex_rings(c, vf_ptr, vf_idx, vv_ptr, vv_idx);
    if (rc == B2TEX_OK) rc = b2tex_set_labels(c, labels);
    if (rc == B2TEX_OK && do_global) rc = b2tex_seam_run(c, si);
    if (rc == B2TEX_OK) rc = b2tex_texture_patches_run(c, do_global ? 1 : 0, pi);
    if (rc == B2TEX_OK && do_local) rc = b2tex_local_seam_leveling_run(c, li);
    if (rc == B2TEX_OK) {
        const size_t n = pi->num_patches, T = pi->num_faces, P = pi->num_pixels;
        *desc_out = (int32_t *)malloc(sizeof(int32_t) * 8 * (n ? n : 1));
        *faces_out = (uint32_t *)malloc(sizeof(uint32_t) * (T ? T : 1));
        *texcoords_out = (float *)malloc(sizeof(float) * 6 * (T ? T : 1));
        *images_out = (float *)malloc(sizeof(float) * 3 * (P ? P : 1));
        *validity_out = (uint8_t *)malloc(P ? P : 1);
        rc = b2tex_texture_patches_download(c, *desc_out, *faces_out, *texcoords_out, *images_out, *validity_out, nullptr);
        if (rc != B2TEX_OK) {   // nothing half-filled leaves the library
            free(*desc_out); free(*faces_out); free(*texcoords_out); free(*images_out); free(*validity_out);
            *desc_out = nullptr; *faces_out = nullptr; *texcoords_out = nullptr; *images_out = nullptr; *validity_out = nullptr;
        }
    }
    release_ctx(c, rc);
    return rc;
}

int b2tex_texture_hot_path(const float *verts, uint32_t nv, const uint32_t *faces, const float *normals, uint32_t nf,
                           const b2tex_view *views, uint32_t K, const uint32_t *adj_ptr, const uint32_t *adj_idx,
                           const uint32_t *vf_ptr, const uint32_t *vf_idx, const uint32_t *vv_ptr,
                           const uint32_t *vv_idx, const b2tex_settings *st, const b2tex_mrf_params *mp,
                           uint32_t *labels_out, uint32_t *row_ptr_out, uint32_t **row_label_out, float **x_out,
                           b2tex_dc_info *dci, b2tex_mrf_info *mi, b2tex_seam_info *si)
{
    if (K > 65535u) { set_error("Exeeded maximal number of views"); return B2TEX_ERR_LIMITS; }
    const int derive = topology_nulls("texture_hot_path", {adj_ptr, adj_idx, vf_ptr, vf_idx, vv_ptr, vv_idx});
    if (derive < 0) return B2TEX_ERR_ARG;
    b2tex_ctx *c = nullptr;
    B2_TRY(acquire_ctx(&c));
    b2tex_dc_info dc_local; b2tex_mrf_info mrf_local; b2tex_seam_info seam_local;
    if (!dci) dci = &dc_local;
    if (!mi) mi = &mrf_local;
    if (!si) si = &seam_local;
    // mesh first (small), then the images on the copy stream: BVH build, culling and the visibility rays of the data-cost
    // stage need no pixels and run while the 1.2 GB (C3) of images are still crossing PCIe
    int rc = b2tex_set_mesh(c, verts, nv, faces, normals, nf);
    c->defer_image_sync = true;
    if (rc == B2TEX_OK) rc = b2tex_set_views(c, views, K);
    c->defer_image_sync = false;
    if (rc == B2TEX_OK && derive) rc = b2tex_build_mesh_graph(c, nullptr);   // runs while the images cross PCIe
    if (rc == B2TEX_OK && !derive) rc = b2tex_set_adjacency(c, adj_ptr, adj_idx);
    if (rc == B2TEX_OK && !derive) rc = b2tex_set_vertex_rings(c, vf_ptr, vf_idx, vv_ptr, vv_idx);
    if (rc == B2TEX_OK) rc = b2tex_data_costs_run(c, st, dci);
    if (c->images_in_flight) { cudaStreamSynchronize(c->copy_stream); c->images_in_flight = false; }   // also on the error paths
    if (rc == B2TEX_OK) rc = b2tex_view_selection_run(c, mp, mi, nullptr);
    if (rc == B2TEX_OK && labels_out) rc = b2tex_labels_download(c, labels_out);
    if (rc == B2TEX_OK) rc = b2tex_seam_run(c, si);
    if (rc == B2TEX_OK && row_ptr_out && row_label_out && x_out) {
        *row_label_out = (uint32_t *)malloc(sizeof(uint32_t) * (si->num_rows ? si->num_rows : 1));
        *x_out = (float *)malloc(sizeof(float) * 3 * (si->num_rows ? si->num_rows : 1));
        rc = b2tex_seam_download(c, row_ptr_out, *row_label_out, *x_out, nullptr);
    }
    release_ctx(c, rc);
    return rc;
}

}  // extern "C"
