// patches.cu -- K10: texture patches and their colour adjustment on the device.
//
// Replaces tex::generate_texture_patches for seen faces (libs/tex/generate_texture_patches.cpp:78-138,453-538;
// hole filling :140-451 is not built) and TexturePatch::adjust_colors (libs/tex/texture_patch.cpp:41-116) as
// driven by global_seam_leveling.cpp:293-323 / texrecon.cpp:174-183.
//
//   host   : label components in the reference's BFS order, candidate merge (patches_host.h)
//   k_project    : pixel coordinates of every face corner in the view of its label + integer bounds per component
//   k_texcoords  : patch-relative texcoords (own candidate origin, then the chain of merge offsets)
//   k_crop       : patch image = crop of the view (magenta outside), bytes / 255          (:126-128)
//   k_adjust_values : per face corner the solved offset of (vertex, label)          (global_seam_leveling.cpp:313-319)
//   k_raster_keys   : one thread per patch triangle; every pixel of its padded box gets a key by atomicMax
//   k_apply         : one thread per pixel; decodes the winning triangle, interpolates, adds, writes the masks
//
// adjust_colors is a sequential loop in which later triangles overwrite earlier ones and "near outside" pixels are
// only written while the pixel is still invalid.  Per pixel that reduces to: if any triangle contains it, the LAST
// such triangle wins (blending 255); otherwise the FIRST triangle within sqrt(2) wins (blending 64).  The key
// (inside: 0x80000000 | index, near: 0x7FFFFFFF - index) makes atomicMax pick exactly that triangle, so the
// result is independent of the execution order and identical to the sequential loop.
#include <math.h>

#include <memory>

#include "patches.cuh"

namespace b2 {

namespace {

// texture_view.h:161-166 with MVE's inner_product order (same restatement as datacosts.cu / seam.cu)
__device__ __forceinline__ void pixel_coords(const ViewDev &V, const float *X, float *out)
{
    float cam[3];
    for (int i = 0; i < 3; ++i)
        cam[i] = (((0.0f + V.w2c[4 * i] * X[0]) + V.w2c[4 * i + 1] * X[1]) + V.w2c[4 * i + 2] * X[2]) + 1.0f * V.w2c[4 * i + 3];
    float pix[3];
    for (int i = 0; i < 3; ++i)
        pix[i] = ((0.0f + V.proj[3 * i] * cam[0]) + V.proj[3 * i + 1] * cam[1]) + V.proj[3 * i + 2] * cam[2];
    out[0] = pix[0] / pix[2] - 0.5f;
    out[1] = pix[1] / pix[2] - 0.5f;
}

// generate_candidate :90-100: one thread per slot (component order)
__global__ void __launch_bounds__(256) k_project(uint32_t T, const uint32_t *__restrict__ comp_faces,
                                                 const uint32_t *__restrict__ slot_comp0, const uint32_t *__restrict__ labels,
                                                 const float *__restrict__ verts, const uint32_t *__restrict__ faces,
                                                 const ViewDev *__restrict__ views, float *px, int32_t *comp_bbox)
{
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= T) return;
    const uint32_t f = comp_faces[s], c = slot_comp0[s];
    const ViewDev &V = views[labels[f] - 1u];
    for (int j = 0; j < 3; ++j) {
        float p[2];
        pixel_coords(V, verts + 3 * (size_t)faces[3 * (size_t)f + j], p);
        px[6 * (size_t)s + 2 * j] = p[0];
        px[6 * (size_t)s + 2 * j + 1] = p[1];
        atomicMin(&comp_bbox[4 * (size_t)c + 0], (int)floorf(p[0]));
        atomicMin(&comp_bbox[4 * (size_t)c + 1], (int)floorf(p[1]));
        atomicMax(&comp_bbox[4 * (size_t)c + 2], (int)ceilf(p[0]));
        atomicMax(&comp_bbox[4 * (size_t)c + 3], (int)ceilf(p[1]));
    }
}

__global__ void k_bbox_init(uint32_t C, const uint32_t *__restrict__ comp_label_view_wh /* [C][2] = W, H */, int32_t *comp_bbox)
{
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    comp_bbox[4 * (size_t)c + 0] = (int32_t)comp_label_view_wh[2 * (size_t)c];      // min_x = width  (:83)
    comp_bbox[4 * (size_t)c + 1] = (int32_t)comp_label_view_wh[2 * (size_t)c + 1];  // min_y = height
    comp_bbox[4 * (size_t)c + 2] = 0;
    comp_bbox[4 * (size_t)c + 3] = 0;
}

// :119-124 (own candidate) and :495-499 (every later merge adds the difference of the origins)
__global__ void __launch_bounds__(256) k_texcoords(uint32_t T, const uint32_t *__restrict__ slot_src,
                                                   const uint32_t *__restrict__ slot_comp, const int32_t *__restrict__ comp_min,
                                                   const uint32_t *__restrict__ comp_chain, const float *__restrict__ chain,
                                                   const float *__restrict__ px, float *tex)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const uint32_t s = slot_src[t], c = slot_comp[t];
    const float mx = (float)comp_min[2 * (size_t)c], my = (float)comp_min[2 * (size_t)c + 1];
    const uint32_t cb = comp_chain[2 * (size_t)c], cn = comp_chain[2 * (size_t)c + 1];
    for (int j = 0; j < 3; ++j) {
        float x = px[6 * (size_t)s + 2 * j] - mx, y = px[6 * (size_t)s + 2 * j + 1] - my;
        for (uint32_t k = 0; k < cn; ++k) { x = x + chain[2 * (size_t)(cb + k)]; y = y + chain[2 * (size_t)(cb + k) + 1]; }
        tex[6 * (size_t)t + 2 * j] = x;
        tex[6 * (size_t)t + 2 * j + 1] = y;
    }
}

// patch of a pixel by binary search in the pixel offsets
__device__ __forceinline__ uint32_t patch_of_pixel(const uint64_t *__restrict__ pix_off, uint32_t n, uint64_t p)
{
    uint32_t lo = 0, hi = n;  // pix_off[lo] <= p < pix_off[hi]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (pix_off[mid] <= p) lo = mid; else hi = mid;
    }
    return lo;
}

// mve::image::crop with fill colour (255,0,255) + byte_to_float_image (:126-128); also clears the raster keys
__global__ void __launch_bounds__(256) k_crop(uint64_t P, uint32_t num_patches, const uint64_t *__restrict__ pix_off,
                                              const int32_t *__restrict__ desc, const ViewDev *__restrict__ views, float *img,
                                              uint32_t *key)
{
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const uint32_t q = patch_of_pixel(pix_off, num_patches, p);
    const int32_t *d = desc + 8 * (size_t)q;
    const uint64_t local = p - pix_off[q];
    const int x = (int)(local % (uint64_t)d[3]), y = (int)(local / (uint64_t)d[3]);
    const ViewDev &V = views[d[0] - 1];
    const int sx = x + d[1], sy = y + d[2];
    uint8_t rgb[3] = {255, 0, 255};
    if (sx >= 0 && sx < V.w && sy >= 0 && sy < V.h) {
        const uint8_t *s = V.rgb + 3 * ((size_t)sx + (size_t)sy * V.w);
        rgb[0] = s[0]; rgb[1] = s[1]; rgb[2] = s[2];
    }
    img[3 * p + 0] = (float)rgb[0] / 255.0f;
    img[3 * p + 1] = (float)rgb[1] / 255.0f;
    img[3 * p + 2] = (float)rgb[2] / 255.0f;
    key[p] = 0u;
}

// adjust_values[vertex].find(label)->second (global_seam_leveling.cpp:313-319); zero when leveling is off
__global__ void __launch_bounds__(256) k_adjust_values(uint32_t T, const uint32_t *__restrict__ slot_face,
                                                       const uint32_t *__restrict__ slot_patch, const int32_t *__restrict__ desc,
                                                       const uint32_t *__restrict__ faces, const uint32_t *__restrict__ row_ptr,
                                                       const uint32_t *__restrict__ row_label, const float *__restrict__ x /* [3][R] */,
                                                       uint32_t R, float *adj /* [T][3][3] */)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const uint32_t f = slot_face[t];
    const uint32_t label = (uint32_t)desc[8 * (size_t)slot_patch[t]];
    for (int j = 0; j < 3; ++j) {
        float a[3] = {0.0f, 0.0f, 0.0f};
        if (x) {
            const uint32_t v = faces[3 * (size_t)f + j];
            for (uint32_t r = row_ptr[v]; r < row_ptr[v + 1]; ++r)
                if (row_label[r] == label) { a[0] = x[r]; a[1] = x[(size_t)R + r]; a[2] = x[2 * (size_t)R + r]; break; }
        }
        adj[9 * (size_t)t + 3 * j + 0] = a[0];
        adj[9 * (size_t)t + 3 * j + 1] = a[1];
        adj[9 * (size_t)t + 3 * j + 2] = a[2];
    }
}

struct PatchTri { float v1x, v1y, v2x, v2y, v3x, v3y, detT, area; };

// Tri::Tri (tri.cpp:12-24) and Tri::get_area (tri.h:78-84)
__device__ __forceinline__ PatchTri make_tri(const float *t6)
{
    PatchTri t;
    t.v1x = t6[0]; t.v1y = t6[1]; t.v2x = t6[2]; t.v2y = t6[3]; t.v3x = t6[4]; t.v3y = t6[5];
    const float T0 = t.v1x - t.v3x, T1 = t.v2x - t.v3x, T2 = t.v1y - t.v3y, T3 = t.v2y - t.v3y;
    t.detT = T0 * T3 - T2 * T1;
    const float u0 = t.v2x - t.v1x, u1 = t.v2y - t.v1y, w0 = t.v3x - t.v1x, w1 = t.v3y - t.v1y;
    t.area = 0.5f * fabsf(u0 * w1 - u1 * w0);
    return t;
}
// Tri::get_barycentric_coords (tri.h:50-56)
__device__ __forceinline__ void bary(const PatchTri &t, float x, float y, float *b)
{
    b[0] = ((t.v2y - t.v3y) * (x - t.v3x) + (t.v3x - t.v2x) * (y - t.v3y)) / t.detT;
    b[1] = ((t.v3y - t.v1y) * (x - t.v3x) + (t.v1x - t.v3x) * (y - t.v3y)) / t.detT;
    b[2] = 1.0f - b[0] - b[1];
}
// 0 = not written, 1 = inside (:71), 2 = within sqrt(2) of the triangle (:85-92)
__device__ __forceinline__ int classify(const PatchTri &t, const float *b)
{
    if (fminf(b[0], fminf(b[1], b[2])) >= 0.0f) return 1;
    const float sqrt_2 = 1.41421354f;  // const float sqrt_2 = sqrt(2)  (texture_patch.cpp:39)
    float dx = t.v2x - t.v3x, dy = t.v2y - t.v3y;
    const float ha = 2.0f * -b[0] * t.area / sqrtf((0.0f + dx * dx) + dy * dy);
    dx = t.v1x - t.v3x; dy = t.v1y - t.v3y;
    const float hb = 2.0f * -b[1] * t.area / sqrtf((0.0f + dx * dx) + dy * dy);
    dx = t.v1x - t.v2x; dy = t.v1y - t.v2y;
    const float hc = 2.0f * -b[2] * t.area / sqrtf((0.0f + dx * dx) + dy * dy);
    if (ha > sqrt_2 || hb > sqrt_2 || hc > sqrt_2) return 0;
    return 2;
}

// texture_patch.cpp:47-96, first half: which triangle writes which pixel
__global__ void __launch_bounds__(256) k_raster_keys(uint32_t T, const uint32_t *__restrict__ slot_patch,
                                                     const int32_t *__restrict__ desc, const uint64_t *__restrict__ pix_off,
                                                     const float *__restrict__ tex, uint32_t *key)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const uint32_t q = slot_patch[t];
    const int32_t *d = desc + 8 * (size_t)q;
    const uint32_t local = t - (uint32_t)d[5];  // index of the triangle inside its patch
    const PatchTri tri = make_tri(tex + 6 * (size_t)t);
    if (tri.area < 1.1920928955078125e-07f) return;  // :53
    const float ax0 = fminf(tri.v1x, fminf(tri.v2x, tri.v3x)), ay0 = fminf(tri.v1y, fminf(tri.v2y, tri.v3y));
    const float ax1 = fmaxf(tri.v1x, fmaxf(tri.v2x, tri.v3x)), ay1 = fmaxf(tri.v1y, fmaxf(tri.v2y, tri.v3y));
    int min_x = (int)floorf(ax0) - PATCH_BORDER, min_y = (int)floorf(ay0) - PATCH_BORDER;
    int max_x = (int)ceilf(ax1) + PATCH_BORDER, max_y = (int)ceilf(ay1) + PATCH_BORDER;
    const int w = d[3], h = d[4];
    // the reference asserts 0 <= min and max <= size (:61-62); stay inside the patch whatever happens
    min_x = max(min_x, 0); min_y = max(min_y, 0); max_x = min(max_x, w); max_y = min(max_y, h);
    uint32_t *k = key + pix_off[q];
    for (int y = min_y; y < max_y; ++y)
        for (int x = min_x; x < max_x; ++x) {
            float b[3];
            bary(tri, (float)x, (float)y, b);
            const int cls = classify(tri, b);
            if (cls == 0) continue;
            const uint32_t kv = cls == 1 ? (0x80000000u | local) : (0x7FFFFFFFu - local);
            atomicMax(&k[(size_t)x + (size_t)y * w], kv);
        }
}

// second half of :47-96 and :98-109: interpolate the winner's adjust values, add them, write the masks
__global__ void __launch_bounds__(256) k_apply(uint64_t P, uint32_t num_patches, const uint64_t *__restrict__ pix_off,
                                               const int32_t *__restrict__ desc, const float *__restrict__ tex,
                                               const float *__restrict__ adj, const uint32_t *__restrict__ key, float *img,
                                               uint8_t *valid, uint8_t *blend)
{
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const uint32_t kv = key[p];
    if (kv == 0u) {  // :104-108
        img[3 * p] = 0.0f; img[3 * p + 1] = 0.0f; img[3 * p + 2] = 0.0f;
        valid[p] = 0; blend[p] = 0;
        return;
    }
    const uint32_t q = patch_of_pixel(pix_off, num_patches, p);
    const int32_t *d = desc + 8 * (size_t)q;
    const uint64_t lp = p - pix_off[q];
    const int x = (int)(lp % (uint64_t)d[3]), y = (int)(lp / (uint64_t)d[3]);
    const bool inside = (kv >> 31) != 0u;
    const uint32_t local = inside ? (kv & 0x7FFFFFFFu) : (0x7FFFFFFFu - kv);
    const size_t t = (size_t)d[5] + local;
    const PatchTri tri = make_tri(tex + 6 * t);
    float b[3];
    bary(tri, (float)x, (float)y, b);
    const float *a = adj + 9 * t;
    for (int c = 0; c < 3; ++c) {
        const float iadj = a[c] * b[0] + a[3 + c] * b[1] + a[6 + c] * b[2];  // math::interpolate, left to right
        img[3 * p + c] = img[3 * p + c] + iadj;
    }
    valid[p] = 255;
    blend[p] = inside ? 255 : 64;
}

}  // namespace

void patches_free(b2tex_ctx *c)
{
    delete c->patches;
    c->patches = nullptr;
}

int patches_run(b2tex_ctx *c, int apply_adjust, b2tex_patch_info *info)
{
    invalidate(c, PATCHES);
    if (!c->F || !c->K) { set_error("texture patches: mesh, views, adjacency and labels must be set"); return B2TEX_ERR_ARG; }
    B2_TRY(require(c, MESH | PIXELS | ADJ | LABELS, "texture patches"));
    if (apply_adjust) B2_TRY(require(c, SEAM, "texture patches with apply_adjust (or pass apply_adjust = 0)"));
    cudaStream_t s = c->stream;
    B2_TRY(prepare_images(c, (c->valid & IMAGES) ? c->prepared_data_term : 0));
    if (!c->patches) c->patches = new PatchState();
    PatchState &ps = *c->patches;
    ps.leveled = false;
    ScopedTimer tm(c, "texture_patches");

    // ---- components on the host (graph traversal, order defining) ----
    std::unique_ptr<ScopedTimer> t_host(new ScopedTimer(c, "tp.download+components"));
    const uint32_t F = c->F;
    std::vector<uint32_t> labels(F), adj_ptr((size_t)F + 1);
    B2_TRY(c->labels.download(labels.data(), F, s));
    B2_TRY(c->adj_ptr.download(adj_ptr.data(), (size_t)F + 1, s));
    B2_CUDA(cudaStreamSynchronize(s));
    std::vector<uint32_t> adj_idx(adj_ptr[F] ? adj_ptr[F] : 1);
    B2_TRY(c->adj_idx.download(adj_idx.data(), adj_ptr[F], s));
    B2_CUDA(cudaStreamSynchronize(s));
    for (uint32_t f = 0; f < F; ++f)
        if (labels[f] > c->K) { set_error("Incorrect labeling"); return B2TEX_ERR_LABELING; }
    std::vector<uint32_t> comp_faces;
    std::vector<PatchComponent> comps;
    label_components(F, adj_ptr.data(), adj_idx.data(), labels.data(), comp_faces, comps);
    const uint32_t T = (uint32_t)comp_faces.size(), C = (uint32_t)comps.size();
    std::vector<uint32_t> slot_comp0(T ? T : 1), comp_wh(2 * (size_t)(C ? C : 1));
    for (uint32_t k = 0; k < C; ++k) {
        for (uint32_t i = comps[k].begin; i < comps[k].end; ++i) slot_comp0[i] = k;
        comp_wh[2 * (size_t)k] = (uint32_t)c->views_host[comps[k].label - 1].width;
        comp_wh[2 * (size_t)k + 1] = (uint32_t)c->views_host[comps[k].label - 1].height;
    }

    t_host.reset();
    // ---- projection + integer bounds per component ----
    std::unique_ptr<ScopedTimer> t_proj(new ScopedTimer(c, "tp.upload+project+bbox"));
    B2_TRY(ps.comp_faces.upload(comp_faces.data(), T, s));
    B2_TRY(ps.slot_comp0.upload(slot_comp0.data(), T, s));
    B2_TRY(ps.comp_wh.upload(comp_wh.data(), 2 * (size_t)C, s));
    B2_TRY(ps.comp_bbox.alloc(4 * (size_t)C));
    B2_TRY(ps.px.alloc(6 * (size_t)T));
    if (C) B2_LAUNCH k_bbox_init<<<(C + 255) / 256, 256, 0, s>>>(C, ps.comp_wh.p, ps.comp_bbox.p);
    if (T) B2_LAUNCH k_project<<<(T + 255) / 256, 256, 0, s>>>(T, ps.comp_faces.p, ps.slot_comp0.p, c->labels.p, c->verts.p, c->faces.p,
                                                     c->views_dev.p, ps.px.p, ps.comp_bbox.p);
    B2_KERNEL_CHECK();
    std::vector<int32_t> bbox(4 * (size_t)(C ? C : 1));
    B2_TRY(ps.comp_bbox.download(bbox.data(), 4 * (size_t)C, s));
    B2_CUDA(cudaStreamSynchronize(s));

    t_proj.reset();
    // ---- candidate merge on the host, then the per-slot / per-pixel work on the device ----
    std::unique_ptr<ScopedTimer> t_plan(new ScopedTimer(c, "tp.merge_plan+upload"));
    plan_patches(comps, bbox.data(), ps.plan);
    const PatchPlan &pl = ps.plan;
    const uint32_t NP = pl.num_patches();
    const uint64_t P = pl.pix_off.back();
    ps.total_pixels = P;
    ps.faces.resize(T);
    for (uint32_t t = 0; t < T; ++t) ps.faces[t] = comp_faces[pl.slot_src[t]];
    B2_TRY(ps.slot_src.upload(pl.slot_src.data(), T, s));
    B2_TRY(ps.slot_comp.upload(pl.slot_comp.data(), T, s));
    B2_TRY(ps.slot_patch.upload(pl.slot_patch.data(), T, s));
    B2_TRY(ps.slot_face.upload(ps.faces.data(), T, s));
    B2_TRY(ps.comp_min.upload(pl.comp_min.data(), 2 * (size_t)C, s));
    B2_TRY(ps.comp_chain.upload(pl.comp_chain.data(), 2 * (size_t)C, s));
    B2_TRY(ps.chain.upload(pl.chain.data(), pl.chain.size(), s));
    B2_TRY(ps.desc.upload(pl.desc.data(), pl.desc.size(), s));
    B2_TRY(ps.pix_off.upload(pl.pix_off.data(), pl.pix_off.size(), s));
    B2_TRY(ps.tex.alloc(6 * (size_t)T));
    B2_TRY(ps.adj.alloc(9 * (size_t)T));
    B2_TRY(ps.img.alloc(3 * P));
    B2_TRY(ps.key.alloc(P));
    B2_TRY(ps.valid.alloc(P));
    B2_TRY(ps.blend.alloc(P));
    t_plan.reset();
    ScopedTimer t_px(c, "tp.texcoords+crop+raster+apply");
    if (T) {
        B2_LAUNCH k_texcoords<<<(T + 255) / 256, 256, 0, s>>>(T, ps.slot_src.p, ps.slot_comp.p, ps.comp_min.p, ps.comp_chain.p, ps.chain.p,
                                                    ps.px.p, ps.tex.p);
        B2_LAUNCH k_adjust_values<<<(T + 255) / 256, 256, 0, s>>>(T, ps.slot_face.p, ps.slot_patch.p, ps.desc.p, c->faces.p,
                                                        apply_adjust ? c->row_ptr.p : nullptr, apply_adjust ? c->row_label.p : nullptr,
                                                        apply_adjust ? c->seam_x.p : nullptr, c->R, ps.adj.p);
    }
    if (P) {
        const unsigned pb = (unsigned)((P + 255) / 256);
        B2_LAUNCH k_crop<<<pb, 256, 0, s>>>(P, NP, ps.pix_off.p, ps.desc.p, c->views_dev.p, ps.img.p, ps.key.p);
        if (T) B2_LAUNCH k_raster_keys<<<(T + 255) / 256, 256, 0, s>>>(T, ps.slot_patch.p, ps.desc.p, ps.pix_off.p, ps.tex.p, ps.key.p);
        B2_LAUNCH k_apply<<<pb, 256, 0, s>>>(P, NP, ps.pix_off.p, ps.desc.p, ps.tex.p, ps.adj.p, ps.key.p, ps.img.p, ps.valid.p, ps.blend.p);
    }
    B2_KERNEL_CHECK();
    B2_CUDA(cudaStreamSynchronize(s));
    info->num_patches = NP;
    info->num_faces = T;
    info->num_pixels = P;
    mark_valid(c, PATCHES);
    return B2TEX_OK;
}

int patches_download(b2tex_ctx *c, int32_t *desc, uint32_t *faces, float *texcoords, float *images, uint8_t *validity,
                     uint8_t *blending)
{
    B2_TRY(require(c, PATCHES, "texture_patches_download"));
    PatchState &ps = *c->patches;
    cudaStream_t s = c->stream;
    const size_t T = ps.faces.size();
    if (desc) memcpy(desc, ps.plan.desc.data(), ps.plan.desc.size() * sizeof(int32_t));
    if (faces && T) memcpy(faces, ps.faces.data(), T * sizeof(uint32_t));
    if (texcoords) B2_TRY(ps.tex.download(texcoords, 6 * T, s));
    if (images) B2_TRY(ps.img.download(images, 3 * ps.total_pixels, s));
    if (validity) B2_TRY(ps.valid.download(validity, ps.total_pixels, s));
    if (blending) B2_TRY(ps.blend.download(blending, ps.total_pixels, s));
    B2_CUDA(cudaStreamSynchronize(s));
    return B2TEX_OK;
}

}  // namespace b2
