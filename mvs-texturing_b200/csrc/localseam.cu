// localseam.cu -- K11: local seam leveling on the device-resident texture patches.
//
// Replaces tex::local_seam_leveling (libs/tex/local_seam_leveling.cpp:105-204) with TexturePatch::
// prepare_blending_mask (texture_patch.cpp:197-297), TexturePatch::blend (:180-192) and poisson_blend
// (poisson_blending.cpp:49-138).  Runs after patches_run() on the patches it left on the device.
//
//   k_seam_edges, k_plan_edges, k_plan_samples, k_plan_vertices : seam edges, their projections into the patches, sampling
//                     density, multi-patch vertices -- from the vertex -> face rings by count / scan / fill, the arrays
//                     the host bookkeeping of patches_host.h produces, element for element (that code remains as the
//                     path for > 16 patches around one vertex and as the cross-check of the emulation tests)
//   k_edge_colors   : mean colour over the adjacent patches at every sample of every seam edge     (:20-37,:131-141)
//   k_vertex_colors : mean colour of every vertex that lies in more than one patch                 (:155-168)
//   k_stamp_keys / k_stamp_apply : vertex pixels, then Bresenham lines (:39-92), written with "last writer wins"
//                     as in the sequential loops :186-193 -- atomicMax on the write order, then one pass that
//                     recomputes the colour of the winning write
//   k_layer_init / k_layer_step x20 / k_sanitize / k_mask_final : prepare_blending_mask as a breadth-first layering
//                     of the valid area (layer k = pixels removed in erosion round k; layer 21 = the new border)
//   k_unknowns, scan, k_poisson_setup, k_poisson_cg, k_poisson_write : poisson_blend with alpha = 1.  The reference
//                     factorises the 5-point system per patch with SparseLU; here ALL patches are solved together by
//                     one persistent cooperative CG on the correction v = u - src (Laplace(v) = 0 inside, v = dest - src
//                     on the Dirichlet pixels), stencil applied on the fly, 3 channels in a float4.  Same system,
//                     iterative instead of direct: results agree to the CG tolerance (1e-5 relative residual).
#include <cooperative_groups.h>
#include <math.h>

#include <memory>

#include "patches.cuh"

namespace cg = cooperative_groups;

namespace b2 {

namespace {

constexpr int STRIP_SIZE = 20;  // local_seam_leveling.cpp:18

__device__ __forceinline__ uint32_t lpatch_of_pixel(const uint64_t *__restrict__ pix_off, uint32_t n, uint64_t p)
{
    uint32_t lo = 0, hi = n;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (pix_off[mid] <= p) lo = mid; else hi = mid;
    }
    return lo;
}

// TexturePatch::get_pixel_value = mve::FloatImage::linear_at on the patch image (texture_patch.cpp:162-169)
__device__ __forceinline__ void patch_linear_at(const float *__restrict__ img, int w, int h, float x, float y, float *out)
{
    x = fmaxf(0.0f, fminf((float)(w - 1), x));
    y = fmaxf(0.0f, fminf((float)(h - 1), y));
    const int fx = (int)x, fy = (int)y;
    const int fx1 = min(fx + 1, w - 1), fy1 = min(fy + 1, h - 1);
    const float w1 = x - (float)fx, w0 = 1.0f - w1;
    const float w3 = y - (float)fy, w2 = 1.0f - w3;
    const float *a = img + 3 * ((size_t)fx + (size_t)fy * w), *b = img + 3 * ((size_t)fx1 + (size_t)fy * w);
    const float *c = img + 3 * ((size_t)fx + (size_t)fy1 * w), *d = img + 3 * ((size_t)fx1 + (size_t)fy1 * w);
    for (int k = 0; k < 3; ++k) out[k] = ((a[k] * (w0 * w2) + b[k] * (w1 * w2)) + c[k] * (w0 * w3)) + d[k] * (w1 * w3);
}


// ---- seam planning on the device -----------------------------------------------------------------------------------
// What patches_host.h does in three passes over host copies (find_seam_edges, vertex_projections, plan_seam_lines:
// downloads and host bookkeeping that dominated this stage) follows from the vertex -> face rings without any sort:
//   * a seam edge (v1 < v2) is projected into exactly the patches that own a face containing the edge (the "common face"
//     test of seam_leveling.cpp:61-91), ascending patch id;
//   * the projection of a vertex into a patch is the texture coordinate of the vertex in the FIRST slot (slots are patch
//     major, in the reference's face order) of that patch that touches it (generate_texture_patches.cpp:520-535: "first
//     projection wins");
//   * a vertex is stamped if faces of more than one patch meet in it (local_seam_leveling.cpp:157).
// Every list is produced by count -> exclusive scan -> fill, so the arrays are the host version's, element for element.
constexpr uint32_t NO_SLOT = 0xFFFFFFFFu;
constexpr int PLAN_MAXP = 16;   // distinct patches around one edge / vertex handled here (more: limit flag -> host path)

struct SeamPlanIn {
    const uint32_t *faces;        // [F][3]
    const uint32_t *vf_ptr, *vf_idx;
    const uint32_t *face_slot;    // [F] final slot of a face, NO_SLOT if it is in no patch
    const uint32_t *slot_patch, *slot_face;
    const float *tex;             // [slots][3][2]
};

__global__ void __launch_bounds__(256) k_face_slot(uint32_t T, const uint32_t *__restrict__ slot_face, uint32_t *face_slot)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < T) face_slot[slot_face[t]] = t;
}

// find_seam_edges (seam_leveling.cpp:16-59): one edge (v1 < v2) per pair of adjacent faces with different labels, face major
template <bool FILL>
__global__ void __launch_bounds__(256) k_seam_edges(uint32_t F, const uint32_t *__restrict__ adj_ptr, const uint32_t *__restrict__ adj_idx,
                                                    const uint32_t *__restrict__ labels, const uint32_t *__restrict__ faces,
                                                    uint32_t *cnt, const uint32_t *__restrict__ off, uint32_t *edges)
{
    const uint32_t node = blockIdx.x * blockDim.x + threadIdx.x;
    if (node >= F) return;
    uint32_t n = 0;
    for (uint32_t a = adj_ptr[node]; a < adj_ptr[node + 1]; ++a) {
        const uint32_t adj = adj_idx[a];
        if (node > adj || labels[node] == labels[adj]) continue;
        uint32_t shared[4]; int ns = 0;
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j)
                if (faces[3 * (size_t)node + i] == faces[3 * (size_t)adj + j] && ns < 4) shared[ns++] = faces[3 * (size_t)node + i];
        if (ns != 2 || shared[0] == shared[1]) continue;   // the reference asserts this
        if (FILL) {
            const uint32_t v1 = min(shared[0], shared[1]), v2 = max(shared[0], shared[1]);
            edges[2 * (size_t)(off[node] + n)] = v1; edges[2 * (size_t)(off[node] + n) + 1] = v2;
        }
        ++n;
    }
    if (!FILL) cnt[node] = n;
}

__device__ __forceinline__ bool plan_face_has(const uint32_t *__restrict__ faces, uint32_t f, uint32_t v)
{
    return faces[3 * (size_t)f] == v || faces[3 * (size_t)f + 1] == v || faces[3 * (size_t)f + 2] == v;
}
// ascending list of distinct patches; false when it overflows
__device__ __forceinline__ bool plan_insert(uint32_t *list, uint32_t &n, uint32_t q)
{
    uint32_t k = 0;
    while (k < n && list[k] < q) ++k;
    if (k < n && list[k] == q) return true;
    if (n >= (uint32_t)PLAN_MAXP) return false;
    for (uint32_t i = n; i > k; --i) list[i] = list[i - 1];
    list[k] = q; ++n;
    return true;
}
// texture coordinate of vertex v in the first slot of patch q that touches it
__device__ __forceinline__ void plan_first_proj(const SeamPlanIn &in, uint32_t v, uint32_t q, float *xy)
{
    uint32_t best = NO_SLOT;
    for (uint32_t a = in.vf_ptr[v]; a < in.vf_ptr[v + 1]; ++a) {
        const uint32_t t = in.face_slot[in.vf_idx[a]];
        if (t != NO_SLOT && in.slot_patch[t] == q && t < best) best = t;
    }
    xy[0] = xy[1] = 0.0f;
    if (best == NO_SLOT) return;
    const uint32_t f = in.slot_face[best];
    const int j = in.faces[3 * (size_t)f] == v ? 0 : (in.faces[3 * (size_t)f + 1] == v ? 1 : 2);
    xy[0] = in.tex[6 * (size_t)best + 2 * j]; xy[1] = in.tex[6 * (size_t)best + 2 * j + 1];
}

// find_mesh_edge_projections (seam_leveling.cpp:61-91) + the sampling density of local_seam_leveling.cpp:131-140, per seam edge.
// count pass: cnt_proj[e], cnt_samp[e]; fill pass: edge_info, proj_patch | proj_edge, edge_proj
template <bool FILL>
__global__ void __launch_bounds__(128) k_plan_edges(uint32_t NE, SeamPlanIn in, const uint32_t *__restrict__ edges, uint32_t *cnt_proj,
                                                    uint32_t *cnt_samp, const uint32_t *__restrict__ off_proj, const uint32_t *__restrict__ off_samp,
                                                    uint32_t NL, uint32_t *edge_info, uint32_t *proj_pack, float *edge_proj, uint32_t *limit_flags)
{
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= NE) return;
    const uint32_t v1 = edges[2 * (size_t)e], v2 = edges[2 * (size_t)e + 1];
    uint32_t list[PLAN_MAXP], n = 0;
    for (uint32_t a = in.vf_ptr[v1]; a < in.vf_ptr[v1 + 1]; ++a) {
        const uint32_t f = in.vf_idx[a];
        if (!plan_face_has(in.faces, f, v2)) continue;
        const uint32_t t = in.face_slot[f];
        if (t == NO_SLOT) continue;
        if (!plan_insert(list, n, in.slot_patch[t])) atomicOr(limit_flags, 1u);
    }
    float max_length = 1.0f;
    for (uint32_t k = 0; k < n; ++k) {
        float p1[2], p2[2];
        plan_first_proj(in, v1, list[k], p1);
        plan_first_proj(in, v2, list[k], p2);
        const float dx = p1[0] - p2[0], dy = p1[1] - p2[1];
        const float length = sqrtf((0.0f + dx * dx) + dy * dy);
        max_length = fmaxf(max_length, length);
        if (FILL) {
            const size_t o = (size_t)off_proj[e] + k;
            proj_pack[o] = list[k]; proj_pack[(size_t)NL + o] = e;
            edge_proj[4 * o] = p1[0]; edge_proj[4 * o + 1] = p1[1]; edge_proj[4 * o + 2] = p2[0]; edge_proj[4 * o + 3] = p2[1];
        }
    }
    const uint32_t ns = (uint32_t)ceilf(max_length * 2.0f);   // :139
    if (FILL) {
        edge_info[4 * (size_t)e] = off_proj[e]; edge_info[4 * (size_t)e + 1] = n;
        edge_info[4 * (size_t)e + 2] = off_samp[e]; edge_info[4 * (size_t)e + 3] = ns;
    } else { cnt_proj[e] = n; cnt_samp[e] = ns; }
}

// every colour sample knows its edge
__global__ void __launch_bounds__(256) k_plan_samples(uint32_t NE, const uint32_t *__restrict__ edge_info, uint32_t *sample_edge)
{
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= NE) return;
    const uint32_t b = edge_info[4 * (size_t)e + 2], n = edge_info[4 * (size_t)e + 3];
    for (uint32_t j = 0; j < n; ++j) sample_edge[(size_t)b + j] = e;
}

// vertices in which faces of more than one patch meet (local_seam_leveling.cpp:155-176), ascending vertex id.
// count pass: cnt_vert[v] (0 / 1), cnt_vproj[v]; fill pass: vert_info, vproj_patch | vproj_vert, vert_proj
template <bool FILL>
__global__ void __launch_bounds__(128) k_plan_vertices(uint32_t Vn, SeamPlanIn in, uint32_t *cnt_vert, uint32_t *cnt_vproj,
                                                       const uint32_t *__restrict__ off_vert, const uint32_t *__restrict__ off_vproj, uint32_t NVP,
                                                       uint32_t *vert_info, uint32_t *vproj_pack, float *vert_proj, uint32_t *limit_flags)
{
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= Vn) return;
    uint32_t list[PLAN_MAXP], n = 0;
    for (uint32_t a = in.vf_ptr[v]; a < in.vf_ptr[v + 1]; ++a) {
        const uint32_t t = in.face_slot[in.vf_idx[a]];
        if (t == NO_SLOT) continue;
        if (!plan_insert(list, n, in.slot_patch[t])) atomicOr(limit_flags, 1u);
    }
    if (!FILL) { cnt_vert[v] = n > 1 ? 1u : 0u; cnt_vproj[v] = n > 1 ? n : 0u; return; }
    if (n <= 1) return;
    const uint32_t iv = off_vert[v], b = off_vproj[v];
    vert_info[2 * (size_t)iv] = b; vert_info[2 * (size_t)iv + 1] = n;
    for (uint32_t k = 0; k < n; ++k) {
        float xy[2];
        plan_first_proj(in, v, list[k], xy);
        vproj_pack[(size_t)b + k] = list[k]; vproj_pack[(size_t)NVP + b + k] = iv;
        vert_proj[2 * ((size_t)b + k)] = xy[0]; vert_proj[2 * ((size_t)b + k) + 1] = xy[1];
    }
}

// mean_color_of_edge_point for sample j of its edge (:20-37), one thread per sample
__global__ void __launch_bounds__(256) k_edge_colors(uint32_t S, const uint32_t *__restrict__ sample_edge,
                                                     const uint32_t *__restrict__ edge_info, const uint32_t *__restrict__ proj_patch,
                                                     const float *__restrict__ edge_proj, const int32_t *__restrict__ desc,
                                                     const uint64_t *__restrict__ pix_off, const float *__restrict__ img,
                                                     float *edge_color)
{
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    const uint32_t *info = edge_info + 4 * (size_t)sample_edge[s];
    const uint32_t j = s - info[2], n = info[3];
    const float t = (float)j / (float)(n - 1u);
    float acc[3] = {0.0f, 0.0f, 0.0f}, wsum = 0.0f;
    for (uint32_t k = info[0]; k < info[0] + info[1]; ++k) {
        const uint32_t q = proj_patch[k];
        const float *p = edge_proj + 4 * (size_t)k;
        const float px = p[0] * t + p[2] * (1.0f - t), py = p[1] * t + p[3] * (1.0f - t);   // p1 * t + (1 - t) * p2
        float col[3];
        patch_linear_at(img + 3 * pix_off[q], desc[8 * (size_t)q + 3], desc[8 * (size_t)q + 4], px, py, col);
        for (int c = 0; c < 3; ++c) acc[c] = acc[c] + col[c] * 1.0f;
        wsum = wsum + 1.0f;
    }
    for (int c = 0; c < 3; ++c) edge_color[3 * (size_t)s + c] = acc[c] / wsum;
}

// :155-168, one thread per vertex that has more than one projection
__global__ void __launch_bounds__(256) k_vertex_colors(uint32_t NV, const uint32_t *__restrict__ vert_info,
                                                       const uint32_t *__restrict__ vproj_patch, const float *__restrict__ vert_proj,
                                                       const int32_t *__restrict__ desc, const uint64_t *__restrict__ pix_off,
                                                       const float *__restrict__ img, float *vert_color)
{
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= NV) return;
    float acc[3] = {0.0f, 0.0f, 0.0f}, wsum = 0.0f;
    for (uint32_t k = vert_info[2 * (size_t)v]; k < vert_info[2 * (size_t)v] + vert_info[2 * (size_t)v + 1]; ++k) {
        const uint32_t q = vproj_patch[k];
        float col[3];
        patch_linear_at(img + 3 * pix_off[q], desc[8 * (size_t)q + 3], desc[8 * (size_t)q + 4], vert_proj[2 * (size_t)k],
                        vert_proj[2 * (size_t)k + 1], col);
        for (int c = 0; c < 3; ++c) acc[c] = acc[c] + col[c] * 1.0f;
        wsum = wsum + 1.0f;
    }
    for (int c = 0; c < 3; ++c) vert_color[3 * (size_t)v + c] = acc[c] / wsum;
}

// write order of :186-193: all vertex pixels of a patch, then its lines; keys only ever compete inside one patch
constexpr uint32_t KEY_LINE = 0x40000000u;

// threads [0, NVP): vertex pixels; threads [NVP, NVP + NL): lines (one per edge projection)
__global__ void __launch_bounds__(256) k_stamp_keys(uint32_t NVP, uint32_t NL, const uint32_t *__restrict__ vproj_patch,
                                                    const float *__restrict__ vert_proj, const uint32_t *__restrict__ proj_patch,
                                                    const float *__restrict__ edge_proj, const int32_t *__restrict__ desc,
                                                    const uint64_t *__restrict__ pix_off, uint32_t *key)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < NVP) {
        const uint32_t q = vproj_patch[i];
        const int w = desc[8 * (size_t)q + 3], h = desc[8 * (size_t)q + 4];
        const int x = (int)(vert_proj[2 * (size_t)i] + 0.5f), y = (int)(vert_proj[2 * (size_t)i + 1] + 0.5f);   // Vec2i(Vec2f): truncation
        if (x >= 0 && x < w && y >= 0 && y < h) atomicMax(&key[pix_off[q] + (size_t)x + (size_t)y * w], 1u + i);
        return;
    }
    const uint32_t l = i - NVP;
    if (l >= NL) return;
    const uint32_t q = proj_patch[l];
    const int w = desc[8 * (size_t)q + 3], h = desc[8 * (size_t)q + 4];
    const float *p = edge_proj + 4 * (size_t)l;
    // Line.from / Line.to are Vec2i (truncation of p + 0.5); draw_line rounds those integers again (identity)
    int x = (int)(p[0] + 0.5f), y = (int)(p[1] + 0.5f);
    const int x1 = (int)(p[2] + 0.5f), y1 = (int)(p[3] + 0.5f);
    const int dx = abs(x1 - x), dy = abs(y1 - y);
    const int sx = x < x1 ? 1 : -1, sy = y < y1 ? 1 : -1;
    int err = dx - dy;
    uint32_t *k = key + pix_off[q];
    for (int guard = 0; guard < 1 << 20; ++guard) {
        if (x >= 0 && x < w && y >= 0 && y < h) atomicMax(&k[(size_t)x + (size_t)y * w], KEY_LINE + 1u + l);
        if (x == x1 && y == y1) break;
        const int e2 = 2 * err;
        if (e2 > -dy) { err -= dy; x += sx; }
        if (e2 < dx) { err += dx; y += sy; }
    }
}

// colour of the winning write (set_pixel_value texture_patch.cpp:171-178; draw_line :57-72)
__global__ void __launch_bounds__(256) k_stamp_apply(uint64_t P, uint32_t num_patches, const uint64_t *__restrict__ pix_off,
                                                     const int32_t *__restrict__ desc, const uint32_t *__restrict__ key,
                                                     const uint32_t *__restrict__ vproj_vert, const float *__restrict__ vert_color,
                                                     const uint32_t *__restrict__ proj_edge, const float *__restrict__ edge_proj,
                                                     const uint32_t *__restrict__ edge_info, const float *__restrict__ edge_color,
                                                     float *img, uint8_t *blend)
{
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const uint32_t kv = key[p];
    if (kv == 0u) return;
    float col[3];
    if (kv < KEY_LINE) {
        const float *c = vert_color + 3 * (size_t)vproj_vert[kv - 1u];
        col[0] = c[0]; col[1] = c[1]; col[2] = c[2];
    } else {
        const uint32_t l = kv - KEY_LINE - 1u;
        const uint32_t q = lpatch_of_pixel(pix_off, num_patches, p);
        const uint64_t lp = p - pix_off[q];
        const int w = desc[8 * (size_t)q + 3];
        const int x = (int)(lp % (uint64_t)w), y = (int)(lp / (uint64_t)w);
        const float *pr = edge_proj + 4 * (size_t)l;
        const int x0 = (int)(pr[0] + 0.5f), y0 = (int)(pr[1] + 0.5f), x1 = (int)(pr[2] + 0.5f), y1 = (int)(pr[3] + 0.5f);
        float tdx = (float)(x1 - x0), tdy = (float)(y1 - y0);
        const float length = sqrtf(tdx * tdx + tdy * tdy);
        tdx = (float)(x1 - x); tdy = (float)(y1 - y);
        const float t = (length != 0.0f) ? sqrtf(tdx * tdx + tdy * tdy) / length : 0.5f;
        const uint32_t *info = edge_info + 4 * (size_t)proj_edge[l];
        const float *ec = edge_color + 3 * (size_t)info[2];
        const uint32_t n = info[3];
        if (t < 1.0f && n > 1u) {
            const uint32_t idx = (uint32_t)floorf(t * (float)(n - 1u));
            for (int c = 0; c < 3; ++c) col[c] = ec[3 * (size_t)idx + c] * (1.0f - t) + ec[3 * (size_t)(idx + 1u) + c] * t;
        } else {
            for (int c = 0; c < 3; ++c) col[c] = ec[3 * (size_t)(n - 1u) + c];
        }
    }
    img[3 * p] = col[0]; img[3 * p + 1] = col[1]; img[3 * p + 2] = col[2];
    blend[p] = 128;
}

// ---- prepare_blending_mask (texture_patch.cpp:197-297) as a breadth-first layering ------------------------------
// layer 1 = valid pixels on the image border or with an invalid 8-neighbour (:203-227)
__global__ void __launch_bounds__(256) k_layer_init(uint64_t P, uint32_t num_patches, const uint64_t *__restrict__ pix_off,
                                                    const int32_t *__restrict__ desc, const uint8_t *__restrict__ valid, uint8_t *layer)
{
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    uint8_t l = 0;
    if (valid[p] != 0) {
        const uint32_t q = lpatch_of_pixel(pix_off, num_patches, p);
        const uint64_t lp = p - pix_off[q];
        const int w = desc[8 * (size_t)q + 3], h = desc[8 * (size_t)q + 4];
        const int x = (int)(lp % (uint64_t)w), y = (int)(lp / (uint64_t)w);
        if (x == 0 || x == w - 1 || y == 0 || y == h - 1) l = 1;
        else
            for (int j = -1; j <= 1 && !l; ++j)
                for (int i = -1; i <= 1; ++i)
                    if (valid[pix_off[q] + (size_t)(x + i) + (size_t)(y + j) * w] == 0) { l = 1; break; }
    }
    layer[p] = l;
}

// erosion round `it` (:232-262): still valid pixels next to a pixel removed in this round form the next border
__global__ void __launch_bounds__(256) k_layer_step(uint64_t P, uint32_t num_patches, const uint64_t *__restrict__ pix_off,
                                                    const int32_t *__restrict__ desc, const uint8_t *__restrict__ valid, uint8_t *layer,
                                                    int it)
{
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    if (valid[p] != 255 || layer[p] != 0) return;   // inner_pixel == 255 and not yet in a border set
    const uint32_t q = lpatch_of_pixel(pix_off, num_patches, p);
    const uint64_t lp = p - pix_off[q];
    const int w = desc[8 * (size_t)q + 3], h = desc[8 * (size_t)q + 4];
    const int x = (int)(lp % (uint64_t)w), y = (int)(lp / (uint64_t)w);
    for (int j = -1; j <= 1; ++j)
        for (int i = -1; i <= 1; ++i) {
            const int nx = x + i, ny = y + j;
            if (nx < 0 || nx >= w || ny < 0 || ny >= h) continue;
            if (layer[pix_off[q] + (size_t)nx + (size_t)ny * w] == (uint8_t)it) { layer[p] = (uint8_t)(it + 1); return; }
        }
}

// :264-281: a stamped pixel (128) whose four neighbours are all 255 becomes 255.  Two adjacent 128 pixels block each
// other, so no conversion can enable another one: the in-place sequential scan and this parallel pass agree.
__global__ void __launch_bounds__(256) k_sanitize(uint64_t P, uint32_t num_patches, const uint64_t *__restrict__ pix_off,
                                                  const int32_t *__restrict__ desc, uint8_t *blend)
{
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    if (blend[p] != 128) return;
    const uint32_t q = lpatch_of_pixel(pix_off, num_patches, p);
    const uint64_t lp = p - pix_off[q];
    const int w = desc[8 * (size_t)q + 3], h = desc[8 * (size_t)q + 4];
    const int x = (int)(lp % (uint64_t)w), y = (int)(lp / (uint64_t)w);
    if (x < 1 || x >= w - 1 || y < 1 || y >= h - 1) return;
    if (blend[p - 1] == 255 && blend[p + 1] == 255 && blend[p - w] == 255 && blend[p + w] == 255) blend[p] = 255;
}

// :283-296: everything deeper than the strip leaves the mask, the innermost border becomes Dirichlet (128)
__global__ void __launch_bounds__(256) k_mask_final(uint64_t P, const uint8_t *__restrict__ valid, const uint8_t *__restrict__ layer,
                                                    uint8_t *blend)
{
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const uint8_t l = layer[p];
    if (valid[p] == 255 && (l == 0 || l == STRIP_SIZE + 1)) blend[p] = 0;
    if (l == STRIP_SIZE + 1) blend[p] = 128;
}

// ---- poisson_blend (poisson_blending.cpp:49-138), alpha = 1 ----------------------------------------------------
__global__ void __launch_bounds__(256) k_unknowns(uint64_t P, const uint8_t *__restrict__ blend, uint32_t *uflag)
{
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p < P) uflag[p] = blend[p] == 255 ? 1u : 0u;
}

// per unknown: its pixel, the unknown index of its four neighbours (or -1) and the right-hand side
//   4 v_i - sum_{unknown nb} v_nb = sum_{Dirichlet nb} (dest_nb - src_nb)
__global__ void __launch_bounds__(256) k_poisson_setup(uint64_t P, uint32_t num_patches, const uint64_t *__restrict__ pix_off,
                                                       const int32_t *__restrict__ desc, const uint8_t *__restrict__ blend,
                                                       const uint32_t *__restrict__ uidx, const float *__restrict__ img,
                                                       const float *__restrict__ orig, uint32_t n, uint32_t *ulist, int32_t *unb /* [4][n] */,
                                                       float *b /* [3][n] */)
{
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P || blend[p] != 255) return;
    const uint32_t i = uidx[p];
    const uint32_t q = lpatch_of_pixel(pix_off, num_patches, p);
    const uint64_t lp = p - pix_off[q];
    const int w = desc[8 * (size_t)q + 3], h = desc[8 * (size_t)q + 4];
    const int x = (int)(lp % (uint64_t)w), y = (int)(lp / (uint64_t)w);
    ulist[i] = (uint32_t)p;   // P < 2^32 is checked by the host
    const int ox[4] = {0, -1, 1, 0}, oy[4] = {-1, 0, 0, 1};
    float rhs[3] = {0.0f, 0.0f, 0.0f};
    for (int k = 0; k < 4; ++k) {
        const int nx = x + ox[k], ny = y + oy[k];
        int32_t ni = -1;
        if (nx >= 0 && nx < w && ny >= 0 && ny < h) {   // the reference asserts that every neighbour is in the mask (:98)
            const uint64_t np = pix_off[q] + (size_t)nx + (size_t)ny * w;
            const uint8_t m = blend[np];
            if (m == 255) ni = (int32_t)uidx[np];
            else if (m == 128 || m == 64)
                for (int c = 0; c < 3; ++c) rhs[c] += img[3 * np + c] - orig[3 * np + c];
        }
        unb[(size_t)k * n + i] = ni;
    }
    for (int c = 0; c < 3; ++c) b[(size_t)c * n + i] = rhs[c];
}

struct PoissonCg {
    uint32_t n;
    const int32_t *unb;     // [4][n]
    const float *b;         // [3][n]
    float *x, *r, *t;       // [3][n]
    float4 *p;              // [n]
    double *partials;       // [2][grid][8]
    uint32_t *status;       // [0..2] iterations, [3..5] residual bits, [6] loop iterations
    uint32_t max_iters;
    float tol;
};

__device__ __forceinline__ void lblock_reduce6(double v[6], double *smem)
{
    for (int k = 0; k < 6; ++k)
        for (int s = 16; s; s >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], s);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0)
        for (int k = 0; k < 6; ++k) smem[warp * 6 + k] = v[k];
    __syncthreads();
    const int nw = blockDim.x >> 5;
    for (int k = 0; k < 6; ++k) {
        double s = 0.0;
        for (int w = 0; w < nw; ++w) s += smem[w * 6 + k];
        v[k] = s;
    }
}
__device__ __forceinline__ void lgrid_totals(const double *part, int nblocks, double out[6], double *smem)
{
    double v[6] = {0, 0, 0, 0, 0, 0};
    for (int b = threadIdx.x; b < nblocks; b += blockDim.x)
        for (int k = 0; k < 6; ++k) v[k] += part[(size_t)b * 8 + k];
    lblock_reduce6(v, smem);
    for (int k = 0; k < 6; ++k) out[k] = v[k];
}

// Conjugate gradients on the 5-point operator (diagonal 4), three right-hand sides at once; same structure as
// k_pcg (seam.cu): fused vector updates, three grid syncs per iteration, deterministic fp64 reductions.
constexpr int LCG_THREADS = 1024;
__global__ void __launch_bounds__(LCG_THREADS, 1) k_poisson_cg(PoissonCg q)
{
    cg::grid_group grid = cg::this_grid();
    __shared__ double smem[(LCG_THREADS / 32) * 6];
    const uint32_t n = q.n;
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
    double *partA = q.partials, *partB = q.partials + (size_t)gridDim.x * 8;
    double acc[6], tot[6];
    for (int k = 0; k < 6; ++k) acc[k] = 0.0;
    for (uint32_t i = tid; i < n; i += nth) {
        float pv[3];
        for (int c = 0; c < 3; ++c) {
            const float rv = q.b[(size_t)c * n + i];
            q.r[(size_t)c * n + i] = rv;
            q.x[(size_t)c * n + i] = 0.0f;
            pv[c] = 0.25f * rv;
            acc[c] += (double)rv * rv;
            acc[3 + c] += (double)rv * pv[c];
        }
        q.p[i] = make_float4(pv[0], pv[1], pv[2], 0.0f);
    }
    lblock_reduce6(acc, smem);
    if (threadIdx.x == 0) for (int k = 0; k < 6; ++k) partA[(size_t)blockIdx.x * 8 + k] = acc[k];
    grid.sync();
    lgrid_totals(partA, gridDim.x, tot, smem);
    float rhsNorm2[3], threshold[3], absNew[3], resNorm2[3];
    bool active[3];
    uint32_t iters[3] = {0, 0, 0};
    for (int c = 0; c < 3; ++c) {
        rhsNorm2[c] = (float)tot[c];
        threshold[c] = q.tol * q.tol * rhsNorm2[c];
        resNorm2[c] = rhsNorm2[c];
        absNew[c] = (float)tot[3 + c];
        active[c] = rhsNorm2[c] != 0.0f && !(resNorm2[c] < threshold[c]);
    }
    uint32_t loops = 0;
    grid.sync();
    while (active[0] || active[1] || active[2]) {
        for (int k = 0; k < 6; ++k) acc[k] = 0.0;
        for (uint32_t i = tid; i < n; i += nth) {   // t = A p, p.t
            const float4 pi = q.p[i];
            float s0 = 4.0f * pi.x, s1 = 4.0f * pi.y, s2 = 4.0f * pi.z;
            for (int k = 0; k < 4; ++k) {
                const int32_t j = q.unb[(size_t)k * n + i];
                if (j >= 0) { const float4 pj = q.p[j]; s0 -= pj.x; s1 -= pj.y; s2 -= pj.z; }
            }
            q.t[i] = s0; q.t[(size_t)n + i] = s1; q.t[2 * (size_t)n + i] = s2;
            acc[0] += (double)pi.x * s0; acc[1] += (double)pi.y * s1; acc[2] += (double)pi.z * s2;
        }
        lblock_reduce6(acc, smem);
        if (threadIdx.x == 0) for (int k = 0; k < 6; ++k) partA[(size_t)blockIdx.x * 8 + k] = acc[k];
        grid.sync();
        lgrid_totals(partA, gridDim.x, tot, smem);
        float alpha[3];
        for (int c = 0; c < 3; ++c) alpha[c] = active[c] ? absNew[c] / (float)tot[c] : 0.0f;
        for (int k = 0; k < 6; ++k) acc[k] = 0.0;
        for (uint32_t i = tid; i < n; i += nth) {   // x += a p, r -= a t, |r|^2, r.z
            const float4 pi = q.p[i];
            const float pv[3] = {pi.x, pi.y, pi.z};
            for (int c = 0; c < 3; ++c) {
                if (!active[c]) continue;
                const size_t o = (size_t)c * n + i;
                q.x[o] += alpha[c] * pv[c];
                const float rv = q.r[o] - alpha[c] * q.t[o];
                q.r[o] = rv;
                acc[c] += (double)rv * rv;
                acc[3 + c] += (double)rv * (0.25f * rv);
            }
        }
        lblock_reduce6(acc, smem);
        if (threadIdx.x == 0) for (int k = 0; k < 6; ++k) partB[(size_t)blockIdx.x * 8 + k] = acc[k];
        grid.sync();
        lgrid_totals(partB, gridDim.x, tot, smem);
        float beta[3] = {0.0f, 0.0f, 0.0f};
        bool upd[3];
        for (int c = 0; c < 3; ++c) {
            upd[c] = false;
            if (!active[c]) continue;
            resNorm2[c] = (float)tot[c];
            if (resNorm2[c] < threshold[c]) { active[c] = false; continue; }
            const float absOld = absNew[c];
            absNew[c] = (float)tot[3 + c];
            beta[c] = absNew[c] / absOld;
            upd[c] = true;
            if (++iters[c] >= q.max_iters) active[c] = false;
        }
        if (upd[0] || upd[1] || upd[2])
            for (uint32_t i = tid; i < n; i += nth) {   // p = z + beta p
                float4 pi = q.p[i];
                if (upd[0]) pi.x = 0.25f * q.r[i] + beta[0] * pi.x;
                if (upd[1]) pi.y = 0.25f * q.r[(size_t)n + i] + beta[1] * pi.y;
                if (upd[2]) pi.z = 0.25f * q.r[2 * (size_t)n + i] + beta[2] * pi.z;
                q.p[i] = pi;
            }
        ++loops;
        grid.sync();
    }
    if (tid == 0) {
        for (int c = 0; c < 3; ++c) {
            q.status[c] = iters[c];
            const float err = rhsNorm2[c] != 0.0f ? sqrtf(resNorm2[c] / rhsNorm2[c]) : 0.0f;
            q.status[3 + c] = __float_as_uint(err);
        }
        q.status[6] = loops;
    }
}

// dest = src + v on the unknowns (:125-136); TexturePatch::blend then invalidates the pixels outside the boundary
// (mask 64, texture_patch.cpp:184-191)
__global__ void __launch_bounds__(256) k_poisson_write(uint64_t P, const uint8_t *__restrict__ blend, const uint32_t *__restrict__ uidx,
                                                       const float *__restrict__ orig, const float *__restrict__ x, uint32_t n, float *img,
                                                       uint8_t *valid)
{
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const uint8_t m = blend[p];
    if (m == 255) {
        const uint32_t i = uidx[p];
        for (int c = 0; c < 3; ++c) img[3 * p + c] = orig[3 * p + c] + x[(size_t)c * n + i];
    } else if (m == 64) {
        valid[p] = 0;
    }
}

}  // namespace

int local_seam_run(b2tex_ctx *c, b2tex_local_seam_info *info)
{
    B2_TRY(require(c, PATCHES, "local seam leveling"));
    PatchState &ps = *c->patches;
    if (ps.leveled) { set_error("local seam leveling was already applied to these patches"); return B2TEX_ERR_ARG; }
    cudaStream_t s = c->stream;
    ScopedTimer tm(c, "local_seam_leveling");
    const PatchPlan &pl = ps.plan;
    const uint32_t NP = pl.num_patches(), T = pl.num_slots(), F = c->F;
    const uint64_t P = ps.total_pixels;
    if (P >= 0xFFFFFFFFull) { set_error("local seam leveling: more than 2^32 patch pixels"); return B2TEX_ERR_LIMITS; }

    // ---- seam planning: seam edges, their projections into the patches, sampling density, multi-patch vertices ----
    DevBuf<uint32_t> &d_sample_edge = ps.sample_edge, &d_edge_info = ps.edge_info, &d_vert_info = ps.vert_info;
    DevBuf<uint32_t> &d_proj = ps.line_info, &d_vproj = ps.pixw_info;   // [proj_patch | proj_edge], [vproj_patch | vproj_vert]
    uint32_t NE = 0, S = 0, NV = 0, NL = 0, NVP = 0;
    static const bool plan_on_host = getenv("B2TEX_LSEAM_HOST") != nullptr;   // diagnostic: the host bookkeeping of patches_host.h
    bool planned = false;
    if ((c->valid & RINGS) && !plan_on_host && T && F < 0x7FFFFFFFu) {
        ScopedTimer t_plan(c, "ls.plan_on_device");
        const uint32_t Vn = c->Vn;
        DevBuf<uint32_t> &face_slot = ps.plan_face_slot, &cnt_a = ps.plan_cnt_a, &cnt_b = ps.plan_cnt_b, &off_a = ps.plan_off_a,
                         &off_b = ps.plan_off_b, &edges = ps.plan_edges, &flags = ps.plan_flags;
        const size_t nmax = (size_t)std::max(F, Vn) + 1;
        B2_TRY(face_slot.alloc(F)); B2_TRY(cnt_a.alloc(nmax)); B2_TRY(cnt_b.alloc(nmax)); B2_TRY(off_a.alloc(nmax)); B2_TRY(off_b.alloc(nmax));
        B2_TRY(flags.alloc(1)); B2_TRY(flags.zero(s));
        B2_CUDA(cudaMemsetAsync(face_slot.p, 0xFF, (size_t)F * sizeof(uint32_t), s));
        B2_LAUNCH k_face_slot<<<(T + 255) / 256, 256, 0, s>>>(T, ps.slot_face.p, face_slot.p);
        // seam edges, face major
        B2_CUDA(cudaMemsetAsync(cnt_a.p, 0, nmax * sizeof(uint32_t), s));
        B2_LAUNCH k_seam_edges<false><<<(F + 255) / 256, 256, 0, s>>>(F, c->adj_ptr.p, c->adj_idx.p, c->labels.p, c->faces.p, cnt_a.p, nullptr, nullptr);
        B2_TRY(cub_exclusive_sum_u32(c, cnt_a.p, off_a.p, (size_t)F + 1));
        B2_CUDA(cudaMemcpyAsync(&NE, off_a.p + F, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        B2_CUDA(cudaStreamSynchronize(s));
        B2_TRY(edges.alloc(2 * (size_t)(NE ? NE : 1)));
        if (NE) B2_LAUNCH k_seam_edges<true><<<(F + 255) / 256, 256, 0, s>>>(F, c->adj_ptr.p, c->adj_idx.p, c->labels.p, c->faces.p, nullptr, off_a.p, edges.p);
        B2_KERNEL_CHECK();
        SeamPlanIn in{c->faces.p, c->vf_ptr.p, c->vf_idx.p, face_slot.p, ps.slot_patch.p, ps.slot_face.p, ps.tex.p};
        // per edge: projections and samples (count -> scan -> fill)
        B2_TRY(cnt_a.alloc(std::max(nmax, (size_t)NE + 1))); B2_TRY(cnt_b.alloc(std::max(nmax, (size_t)NE + 1)));
        B2_TRY(off_a.alloc(std::max(nmax, (size_t)NE + 1))); B2_TRY(off_b.alloc(std::max(nmax, (size_t)NE + 1)));
        B2_CUDA(cudaMemsetAsync(cnt_a.p + NE, 0, sizeof(uint32_t), s));
        B2_CUDA(cudaMemsetAsync(cnt_b.p + NE, 0, sizeof(uint32_t), s));
        if (NE) B2_LAUNCH k_plan_edges<false><<<(NE + 127) / 128, 128, 0, s>>>(NE, in, edges.p, cnt_a.p, cnt_b.p, nullptr, nullptr, 0u, nullptr, nullptr, nullptr, flags.p);
        B2_TRY(cub_exclusive_sum_u32(c, cnt_a.p, off_a.p, (size_t)NE + 1));
        B2_TRY(cub_exclusive_sum_u32(c, cnt_b.p, off_b.p, (size_t)NE + 1));
        uint32_t lim = 0;
        B2_CUDA(cudaMemcpyAsync(&NL, off_a.p + NE, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        B2_CUDA(cudaMemcpyAsync(&S, off_b.p + NE, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        B2_CUDA(cudaMemcpyAsync(&lim, flags.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        B2_CUDA(cudaStreamSynchronize(s));
        if (!lim) {
            B2_TRY(d_edge_info.alloc(4 * (size_t)(NE ? NE : 1))); B2_TRY(d_proj.alloc(2 * (size_t)(NL ? NL : 1)));
            B2_TRY(ps.edge_proj.alloc(4 * (size_t)(NL ? NL : 1))); B2_TRY(d_sample_edge.alloc(S ? S : 1));
            if (NE) {
                B2_LAUNCH k_plan_edges<true><<<(NE + 127) / 128, 128, 0, s>>>(NE, in, edges.p, nullptr, nullptr, off_a.p, off_b.p, NL, d_edge_info.p, d_proj.p,
                                                                    ps.edge_proj.p, flags.p);
                B2_LAUNCH k_plan_samples<<<(NE + 255) / 256, 256, 0, s>>>(NE, d_edge_info.p, d_sample_edge.p);
            }
            // multi-patch vertices
            B2_TRY(cnt_a.alloc(std::max(nmax, (size_t)NE + 1)));
            B2_CUDA(cudaMemsetAsync(cnt_a.p + Vn, 0, sizeof(uint32_t), s));
            B2_CUDA(cudaMemsetAsync(cnt_b.p + Vn, 0, sizeof(uint32_t), s));
            B2_LAUNCH k_plan_vertices<false><<<(Vn + 127) / 128, 128, 0, s>>>(Vn, in, cnt_a.p, cnt_b.p, nullptr, nullptr, 0u, nullptr, nullptr, nullptr, flags.p);
            B2_TRY(cub_exclusive_sum_u32(c, cnt_a.p, off_a.p, (size_t)Vn + 1));
            B2_TRY(cub_exclusive_sum_u32(c, cnt_b.p, off_b.p, (size_t)Vn + 1));
            B2_CUDA(cudaMemcpyAsync(&NV, off_a.p + Vn, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
            B2_CUDA(cudaMemcpyAsync(&NVP, off_b.p + Vn, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
            B2_CUDA(cudaMemcpyAsync(&lim, flags.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
            B2_CUDA(cudaStreamSynchronize(s));
        }
        if (!lim) {
            B2_TRY(d_vert_info.alloc(2 * (size_t)(NV ? NV : 1))); B2_TRY(d_vproj.alloc(2 * (size_t)(NVP ? NVP : 1)));
            B2_TRY(ps.vert_proj.alloc(2 * (size_t)(NVP ? NVP : 1)));
            B2_LAUNCH k_plan_vertices<true><<<(Vn + 127) / 128, 128, 0, s>>>(Vn, in, nullptr, nullptr, off_a.p, off_b.p, NVP, d_vert_info.p, d_vproj.p,
                                                                  ps.vert_proj.p, flags.p);
            B2_KERNEL_CHECK();
            planned = true;
        }
        // more than PLAN_MAXP patches around one edge or vertex: the host bookkeeping below has no such limit
    }
    if (!planned) {
    // ---- host bookkeeping: vertex projections, seam edges and their projections ----
    std::unique_ptr<ScopedTimer> t_host(new ScopedTimer(c, "ls.download+host_bookkeeping"));
    std::vector<float> tex(6 * (size_t)(T ? T : 1));
    std::vector<uint32_t> labels(F), adj_ptr((size_t)F + 1), mesh_faces(3 * (size_t)F);
    B2_TRY(ps.tex.download(tex.data(), 6 * (size_t)T, s));
    B2_TRY(c->labels.download(labels.data(), F, s));
    B2_TRY(c->adj_ptr.download(adj_ptr.data(), (size_t)F + 1, s));
    B2_TRY(c->faces.download(mesh_faces.data(), 3 * (size_t)F, s));
    B2_CUDA(cudaStreamSynchronize(s));
    std::vector<uint32_t> adj_idx(adj_ptr[F] ? adj_ptr[F] : 1);
    B2_TRY(c->adj_idx.download(adj_idx.data(), adj_ptr[F], s));
    B2_CUDA(cudaStreamSynchronize(s));
    std::vector<uint32_t> seam_edges;
    find_seam_edges(F, adj_ptr.data(), adj_idx.data(), labels.data(), mesh_faces.data(), seam_edges);
    VertexProjections vpi;
    vertex_projections(c->Vn, mesh_faces.data(), pl, ps.faces.data(), tex.data(), seam_edges, vpi);
    SeamLines sl;
    plan_seam_lines(seam_edges, vpi, sl);
    NE = sl.num_edges(); S = sl.num_samples(); NV = sl.num_verts();
    NL = (uint32_t)sl.proj_patch.size(); NVP = (uint32_t)sl.vert_proj_patch.size();
    std::vector<uint32_t> proj_edge(NL ? NL : 1), vproj_vert(NVP ? NVP : 1);
    for (uint32_t e = 0; e < NE; ++e)
        for (uint32_t k = sl.edge_info[4 * (size_t)e]; k < sl.edge_info[4 * (size_t)e] + sl.edge_info[4 * (size_t)e + 1]; ++k) proj_edge[k] = e;
    for (uint32_t v = 0; v < NV; ++v)
        for (uint32_t k = sl.vert_info[2 * (size_t)v]; k < sl.vert_info[2 * (size_t)v] + sl.vert_info[2 * (size_t)v + 1]; ++k) vproj_vert[k] = v;
    t_host.reset();
    std::vector<uint32_t> pack(2 * (size_t)(NL ? NL : 1)), vpack(2 * (size_t)(NVP ? NVP : 1));
    for (uint32_t k = 0; k < NL; ++k) { pack[k] = sl.proj_patch[k]; pack[(size_t)NL + k] = proj_edge[k]; }
    for (uint32_t k = 0; k < NVP; ++k) { vpack[k] = sl.vert_proj_patch[k]; vpack[(size_t)NVP + k] = vproj_vert[k]; }
    B2_TRY(d_sample_edge.upload(sl.sample_edge.data(), S, s));
    B2_TRY(d_edge_info.upload(sl.edge_info.data(), 4 * (size_t)NE, s));
    B2_TRY(d_vert_info.upload(sl.vert_info.data(), 2 * (size_t)NV, s));
    B2_TRY(d_proj.upload(pack.data(), 2 * (size_t)NL, s));
    B2_TRY(d_vproj.upload(vpack.data(), 2 * (size_t)NVP, s));
    B2_TRY(ps.edge_proj.upload(sl.edge_proj.data(), 4 * (size_t)NL, s));
    B2_TRY(ps.vert_proj.upload(sl.vert_proj.data(), 2 * (size_t)NVP, s));
    B2_CUDA(cudaStreamSynchronize(s));   // the staging vectors are locals of this block
    }
    // ---- colours, stamping ----
    std::unique_ptr<ScopedTimer> t_col(new ScopedTimer(c, "ls.colors+stamp"));
    B2_TRY(ps.edge_color.alloc(3 * (size_t)S));
    B2_TRY(ps.vert_color.alloc(3 * (size_t)NV));
    B2_TRY(ps.orig.alloc(3 * P));
    B2_TRY(ps.layer.alloc(P));
    const unsigned pb = (unsigned)((P + 255) / 256);
    if (P) B2_CUDA(cudaMemcpyAsync(ps.orig.p, ps.img.p, 3 * P * sizeof(float), cudaMemcpyDeviceToDevice, s));   // :181 duplicate()
    if (S) B2_LAUNCH k_edge_colors<<<(S + 255) / 256, 256, 0, s>>>(S, d_sample_edge.p, d_edge_info.p, d_proj.p, ps.edge_proj.p, ps.desc.p, ps.pix_off.p,
                                                         ps.img.p, ps.edge_color.p);
    if (NV) B2_LAUNCH k_vertex_colors<<<(NV + 255) / 256, 256, 0, s>>>(NV, d_vert_info.p, d_vproj.p, ps.vert_proj.p, ps.desc.p, ps.pix_off.p, ps.img.p,
                                                             ps.vert_color.p);
    B2_KERNEL_CHECK();
    if (P) {
        B2_CUDA(cudaMemsetAsync(ps.key.p, 0, P * sizeof(uint32_t), s));
        if (NVP + NL) B2_LAUNCH k_stamp_keys<<<(NVP + NL + 255) / 256, 256, 0, s>>>(NVP, NL, d_vproj.p, ps.vert_proj.p, d_proj.p, ps.edge_proj.p, ps.desc.p,
                                                                         ps.pix_off.p, ps.key.p);
        B2_LAUNCH k_stamp_apply<<<pb, 256, 0, s>>>(P, NP, ps.pix_off.p, ps.desc.p, ps.key.p, d_vproj.p + NVP, ps.vert_color.p, d_proj.p + NL, ps.edge_proj.p,
                                         d_edge_info.p, ps.edge_color.p, ps.img.p, ps.blend.p);
        t_col.reset();
        // ---- blending mask ----
        ScopedTimer t_mask(c, "ls.blending_mask");
        B2_LAUNCH k_layer_init<<<pb, 256, 0, s>>>(P, NP, ps.pix_off.p, ps.desc.p, ps.valid.p, ps.layer.p);
        for (int it = 1; it <= STRIP_SIZE; ++it) B2_LAUNCH k_layer_step<<<pb, 256, 0, s>>>(P, NP, ps.pix_off.p, ps.desc.p, ps.valid.p, ps.layer.p, it);
        B2_LAUNCH k_sanitize<<<pb, 256, 0, s>>>(P, NP, ps.pix_off.p, ps.desc.p, ps.blend.p);
        B2_LAUNCH k_mask_final<<<pb, 256, 0, s>>>(P, ps.valid.p, ps.layer.p, ps.blend.p);
        B2_KERNEL_CHECK();
    }
    t_col.reset();
    // ---- Poisson blending ----
    ScopedTimer t_poi(c, "ls.poisson");
    uint32_t n = 0;
    uint32_t st[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (P) {
        B2_TRY(ps.uflag.alloc(P + 1));
        B2_TRY(ps.uidx.alloc(P + 1));
        B2_CUDA(cudaMemsetAsync(ps.uflag.p + P, 0, sizeof(uint32_t), s));
        B2_LAUNCH k_unknowns<<<pb, 256, 0, s>>>(P, ps.blend.p, ps.uflag.p);
        B2_TRY(cub_exclusive_sum_u32(c, ps.uflag.p, ps.uidx.p, (size_t)P + 1));
        B2_CUDA(cudaMemcpyAsync(&n, ps.uidx.p + P, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        B2_CUDA(cudaStreamSynchronize(s));
    }
    if (n) {
        B2_TRY(ps.ulist.alloc(n));
        DevBuf<int32_t> &unb = ps.unb;
        B2_TRY(unb.alloc(4 * (size_t)n));
        B2_TRY(ps.cg_b.alloc(3 * (size_t)n)); B2_TRY(ps.cg_x.alloc(3 * (size_t)n));
        B2_TRY(ps.cg_r.alloc(3 * (size_t)n)); B2_TRY(ps.cg_t.alloc(3 * (size_t)n));
        B2_TRY(ps.cg_p.alloc(n));
        B2_TRY(ps.cg_status.alloc(16));
        B2_TRY(ps.cg_status.zero(s));
        B2_LAUNCH k_poisson_setup<<<pb, 256, 0, s>>>(P, NP, ps.pix_off.p, ps.desc.p, ps.blend.p, ps.uidx.p, ps.img.p, ps.orig.p, n, ps.ulist.p,
                                           unb.p, ps.cg_b.p);
        B2_KERNEL_CHECK();
        int per_sm = 0;
        B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_poisson_cg, LCG_THREADS, 0));
        if (per_sm < 1) { set_error("k_poisson_cg cannot be resident"); return B2TEX_ERR_CUDA; }
        int grid = c->num_sms * per_sm;
        const int need = (int)((n + LCG_THREADS - 1) / LCG_THREADS);
        if (grid > need) grid = std::max(1, need);
        B2_TRY(ps.cg_partials.alloc(2 * (size_t)grid * 8));
        PoissonCg q{n, unb.p, ps.cg_b.p, ps.cg_x.p, ps.cg_r.p, ps.cg_t.p, ps.cg_p.p, ps.cg_partials.p,
                    ps.cg_status.p, 2000u, 1e-5f};
        void *args[] = {&q};
        count_launch();
        B2_CUDA(cudaLaunchCooperativeKernel((void *)k_poisson_cg, dim3(grid), dim3(LCG_THREADS), args, 0, s));
        B2_CUDA(cudaMemcpyAsync(st, ps.cg_status.p, sizeof(st), cudaMemcpyDeviceToHost, s));
    }
    if (P) B2_LAUNCH k_poisson_write<<<pb, 256, 0, s>>>(P, ps.blend.p, ps.uidx.p, ps.orig.p, n ? ps.cg_x.p : nullptr, n, ps.img.p, ps.valid.p);
    B2_KERNEL_CHECK();
    B2_CUDA(cudaStreamSynchronize(s));
    ps.leveled = true;
    info->num_seam_edges = NE;
    info->num_edge_samples = S;
    info->num_vertices = NV;
    info->num_unknowns = n;
    for (int ch = 0; ch < 3; ++ch) { info->iterations[ch] = st[ch]; memcpy(&info->residual[ch], &st[3 + ch], 4); }
    return B2TEX_OK;
}

}  // namespace b2
