// datacosts.cu -- K3/K4: per-(face,view) data costs on the device.
//
// Replaces calculate_face_projection_infos + postprocess_face_infos
// (libs/tex/calculate_data_costs.cpp:131-306) and TextureView::get_face_info / inside / valid_pixel
// (libs/tex/texture_view.cpp:134-281, texture_view.h:153-166).  fp32 arithmetic mirrors the
// reference's operation order (compile with -fmad=false); fp64 accumulation of the footprint as in
// texture_view.cpp:157,215,224.
//
// Pipeline (all faces of the context's face range, all views):
//   cull<count>  : back-face / frustum / 75 degree / 3-vertex validity, thread per face -> candidates per
//                  face + one bit per surviving view (pass_bits[face][ceil(K/32)])
//   scan         : candidate offsets (CSR by face)
//   cull<fill>   : candidate (face,view) list + the set of (vertex,view) rays that are needed; warp per face,
//                  lane l of pass word w owns view 32w+l, so the list is written in contiguous runs
//   rays         : ONE visibility ray per needed (vertex,view) -- the reference traces the same ray
//                  once per incident face (calculate_data_costs.cpp:197-213); the result depends only
//                  on (vertex, view), so it is shared (about 6x fewer rays, identical answers)
//   quality      : occlusion lookup + footprint integral (GMI) per candidate, global max
//   count_survivors -> scan -> compact : drop quality==0, CSR by face with ascending views (:222, :272);
//                  the compaction runs warp per face, 32-candidate chunks, prefix popcount of the survivor mask
//   histogram -> percentile -> normalise (:277-302, histogram.cpp:22-63)
#include <cub/cub.cuh>

#include <math.h>

#include "bvh.cuh"
#include "common.cuh"
#include "sampling.cuh"

namespace b2 {

int cub_exclusive_sum_u64(b2tex_ctx *c, const uint64_t *in, uint64_t *out, size_t n)
{
    size_t bytes = 0;
    B2_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, n, c->stream));
    B2_TRY(c->cub_tmp.alloc(bytes));
    B2_CUDA(cub::DeviceScan::ExclusiveSum(c->cub_tmp.p, bytes, in, out, n, c->stream));
    return B2TEX_OK;
}
int cub_exclusive_sum_u32(b2tex_ctx *c, const uint32_t *in, uint32_t *out, size_t n)
{
    size_t bytes = 0;
    B2_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, n, c->stream));
    B2_TRY(c->cub_tmp.alloc(bytes));
    B2_CUDA(cub::DeviceScan::ExclusiveSum(c->cub_tmp.p, bytes, in, out, n, c->stream));
    return B2TEX_OK;
}

namespace {

struct Px { float x, y; };

// texture_view.h:161-166 with MVE's inner_product order
__device__ __forceinline__ Px pixel_coords(const ViewDev &V, const float *X)
{
    float cam[3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
        cam[i] = (((0.0f + V.w2c[4 * i] * X[0]) + V.w2c[4 * i + 1] * X[1]) + V.w2c[4 * i + 2] * X[2])
            + 1.0f * V.w2c[4 * i + 3];
    float pix[3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
        pix[i] = ((0.0f + V.proj[3 * i] * cam[0]) + V.proj[3 * i + 1] * cam[1]) + V.proj[3 * i + 2] * cam[2];
    Px p;
    p.x = pix[0] / pix[2] - 0.5f;
    p.y = pix[1] / pix[2] - 0.5f;
    return p;
}

// texture_view.cpp:253-281
__device__ __forceinline__ bool valid_pixel(const ViewDev &V, Px p)
{
    bool valid = (p.x >= 0.0f && p.x < (float)(V.w - 1) && p.y >= 0.0f && p.y < (float)(V.h - 1));
    if (valid && V.valid4) {
        int fx = (int)p.x, fy = (int)p.y;
        valid = V.valid4[(size_t)fx + (size_t)fy * V.w] != 0;
    }
    return valid;
}

struct FaceGeom { float v[3][3]; float n[3]; float c[3]; };

__device__ __forceinline__ void load_face(const float *__restrict__ verts, const uint32_t *__restrict__ faces,
                                          const float *__restrict__ normals, uint32_t f, FaceGeom &g,
                                          uint32_t vid[3])
{
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        vid[k] = faces[3 * (size_t)f + k];
        g.v[k][0] = verts[3 * (size_t)vid[k]];
        g.v[k][1] = verts[3 * (size_t)vid[k] + 1];
        g.v[k][2] = verts[3 * (size_t)vid[k] + 2];
    }
    if (normals) {
        g.n[0] = normals[3 * (size_t)f]; g.n[1] = normals[3 * (size_t)f + 1]; g.n[2] = normals[3 * (size_t)f + 2];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) g.c[k] = ((g.v[0][k] + g.v[1][k]) + g.v[2][k]) / 3.0f;  // :175
}

// calculate_data_costs.cpp:179-191; returns true if the pair survives culling and projects validly
__device__ __forceinline__ bool cull_pair(const ViewDev &V, const FaceGeom &g, float cos_thr, float margin)
{
    float ftv[3] = {V.pos[0] - g.c[0], V.pos[1] - g.c[1], V.pos[2] - g.c[2]};
    {
        // Conservative pre-rejects on the UNNORMALISED vector (no sqrt, no divisions).  They only fire
        // when the exact test below is certain to fail: `margin` (1e-5 * max(1,|n|)) is > 10x the
        // worst-case rounding difference between dot(ftv/|ftv|, n) and dot(ftv, n)/|ftv|.  Everything
        // else takes the exact path, so the surviving set is unchanged (bit-exact vs the oracle).
        const float d0 = ftv[0] * g.n[0] + ftv[1] * g.n[1] + ftv[2] * g.n[2];
        const float len2 = ftv[0] * ftv[0] + ftv[1] * ftv[1] + ftv[2] * ftv[2];
        const float m2 = margin * margin * len2;
        if (d0 < 0.0f && d0 * d0 > m2) return false;                        // back face (:183-185)
        const float ct = cos_thr - margin;
        if (d0 >= 0.0f && ct > 0.0f && d0 * d0 < ct * ct * len2) return false;  // > 75 degrees (:187)
        const float dd = V.dir[0] * ftv[0] + V.dir[1] * ftv[1] + V.dir[2] * ftv[2];
        const float dir2 = V.dir[0] * V.dir[0] + V.dir[1] * V.dir[1] + V.dir[2] * V.dir[2];
        if (dd > 0.0f && dd * dd > 1e-10f * fmaxf(1.0f, dir2) * len2) return false;  // behind the camera
    }
    float nrm = sqrtf(((0.0f + ftv[0] * ftv[0]) + ftv[1] * ftv[1]) + ftv[2] * ftv[2]);
    ftv[0] = ftv[0] / nrm; ftv[1] = ftv[1] / nrm; ftv[2] = ftv[2] / nrm;
    float viewing_angle = ((0.0f + ftv[0] * g.n[0]) + ftv[1] * g.n[1]) + ftv[2] * g.n[2];
    // view_to_face = -face_to_view exactly, so dot(viewdir, view_to_face) < 0 <=> the negated sum < 0
    float dv = ((0.0f + V.dir[0] * (-ftv[0])) + V.dir[1] * (-ftv[1])) + V.dir[2] * (-ftv[2]);
    if (viewing_angle < 0.0f || dv < 0.0f) return false;
    // std::acos(viewing_angle) > MATH_DEG2RAD(75.0f)  <=>  viewing_angle < cos_thr (host bisection
    // on acosf; NaN for |x|>1 keeps the pair exactly like the reference's false comparison)
    if (viewing_angle < cos_thr) return false;
    Px p1 = pixel_coords(V, g.v[0]);
    if (!valid_pixel(V, p1)) return false;
    Px p2 = pixel_coords(V, g.v[1]);
    if (!valid_pixel(V, p2)) return false;
    Px p3 = pixel_coords(V, g.v[2]);
    return valid_pixel(V, p3);
}

// The candidate kernels run one WARP per face where they touch the candidate list (grid-stride over the faces), so that
// the ~44 candidates of a face are read and written by neighbouring lanes: contiguous runs instead of one thread per face
// striding 44 elements.  A lane gets its slot from a 32-bit mask of the face's current 32 candidates that every lane
// forms itself from the same (broadcast) loads, so the kernels need no warp collective and each lane's work depends on
// nothing but memory: the host emulation (tests/cpp/cuda_emul.h) runs them thread after thread.
__device__ __forceinline__ uint32_t lanemask_lt() { return (1u << (threadIdx.x & 31u)) - 1u; }
__device__ __forceinline__ uint32_t warp_id() { return (blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
__device__ __forceinline__ uint32_t num_warps() { return (gridDim.x * blockDim.x) >> 5; }

// count pass, thread per face, loop over the K views: the surviving views go to pass_bits[f - face_begin][kwords]
// (bit j of word j/32 = view j), their number to cand_cnt[f]
__device__ __forceinline__ void cull_count(const float *__restrict__ verts, const uint32_t *__restrict__ faces,
                                           const float *__restrict__ normals, const ViewDev *__restrict__ views, uint32_t K,
                                           uint32_t face_begin, uint32_t face_end, float cos_thr, uint64_t *cand_cnt,
                                           uint32_t *pass_bits, uint32_t kwords)
{
    uint32_t f = face_begin + blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= face_end) return;
    FaceGeom g;
    uint32_t vid[3];
    load_face(verts, faces, normals, f, g, vid);
    const float margin = 1e-5f * fmaxf(1.0f, sqrtf(g.n[0] * g.n[0] + g.n[1] * g.n[1] + g.n[2] * g.n[2]));
    uint32_t count = 0;
    uint32_t bits = 0;
    for (uint32_t j = 0; j < K; ++j) {
        const bool pass = cull_pair(views[j], g, cos_thr, margin);
        if (pass) bits |= 1u << (j & 31u);
        if ((j & 31u) == 31u || j + 1 == K) { pass_bits[(size_t)(f - face_begin) * kwords + (j >> 5)] = bits; bits = 0; }
        count += pass;
    }
    cand_cnt[f] = count;
}

// fill pass, warp per face: the (face, view) list in CSR order (views ascending) from the pass bits, and the set of
// (vertex, view) rays that are needed.  Lane l of pass word w owns view 32w+l; its slot is the face's offset + the
// candidates of the earlier words + the set bits below l.
__device__ __forceinline__ void cull_fill(const uint32_t *__restrict__ faces, uint32_t face_begin, uint32_t face_end,
                                          const uint64_t *__restrict__ cand_ptr, uint16_t *cand_view, uint32_t *cand_face,
                                          uint32_t *need_bits, uint32_t vwords, const uint32_t *__restrict__ vrank,
                                          const uint32_t *__restrict__ pass_bits, uint32_t kwords)
{
    const uint32_t lane = threadIdx.x & 31u, lt = lanemask_lt();
    for (uint32_t f = face_begin + warp_id(); f < face_end; f += num_warps()) {
        uint64_t o = cand_ptr[f];
        // ray bitmaps are indexed by the Morton rank of the vertex so that a warp of k_rays traces 32 spatially
        // adjacent origins towards the same camera.  Vertices of the face that share a bitmap word share one update.
        uint32_t vw[3] = {0, 0, 0}, vb[3] = {0, 0, 0};
        if (need_bits) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const uint32_t r = vrank[faces[3 * (size_t)f + k]];
                vw[k] = r >> 5; vb[k] = 1u << (r & 31u);
            }
            if (vw[1] == vw[0]) { vb[0] |= vb[1]; vb[1] = 0; }
            if (vw[2] == vw[0]) { vb[0] |= vb[2]; vb[2] = 0; }
            else if (vw[2] == vw[1] && vb[1]) { vb[1] |= vb[2]; vb[2] = 0; }
        }
        const uint32_t *pb = pass_bits + (size_t)(f - face_begin) * kwords;
        for (uint32_t w = 0; w < kwords; ++w) {
            const uint32_t word = pb[w];   // the same address in every lane: one transaction
            if ((word >> lane) & 1u) {
                const uint32_t j = 32u * w + lane;
                const uint64_t slot = o + __popc(word & lt);
                cand_view[slot] = (uint16_t)j;
                cand_face[slot] = f;
                if (need_bits) {
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        if (!vb[k]) continue;
                        uint32_t *p = need_bits + (size_t)j * vwords + vw[k];
                        if ((*p & vb[k]) != vb[k]) atomicOr(p, vb[k]);
                    }
                }
            }
            o += __popc(word);
        }
    }
}

// count: thread per face (launch with >= face_end - face_begin threads); fill: warp per face (any grid)
template <bool FILL>
__global__ void __launch_bounds__(256) k_cull(const float *__restrict__ verts, const uint32_t *__restrict__ faces,
                                              const float *__restrict__ normals, const ViewDev *__restrict__ views,
                                              uint32_t K, uint32_t face_begin, uint32_t face_end, float cos_thr,
                                              uint64_t *cand_cnt, const uint64_t *__restrict__ cand_ptr,
                                              uint16_t *cand_view, uint32_t *cand_face, uint32_t *need_bits,
                                              uint32_t vwords, const uint32_t *__restrict__ vrank,
                                              uint32_t *pass_bits, uint32_t kwords)
{
    if (FILL) cull_fill(faces, face_begin, face_end, cand_ptr, cand_view, cand_face, need_bits, vwords, vrank, pass_bits, kwords);
    else cull_count(verts, faces, normals, views, K, face_begin, face_end, cos_thr, cand_cnt, pass_bits, kwords);
}

// one warp = 32 consecutive vertices of one view; lane 0 publishes the 32 occlusion bits
__global__ void __launch_bounds__(256) k_rays(const float *__restrict__ verts, uint32_t Vn,
                                              const ViewDev *__restrict__ views, uint32_t K,
                                              const uint32_t *__restrict__ need_bits, uint32_t *occ_bits,
                                              uint32_t vwords, const uint32_t *__restrict__ vorder,
                                              const BvhNode *__restrict__ nodes,
                                              const float *__restrict__ tri, uint32_t num_tris,
                                              unsigned long long *ray_count, uint32_t *stack_overflow)
{
    size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    size_t total = (size_t)K * vwords;
    if (warp >= total) return;
    uint32_t lane = threadIdx.x & 31;
    uint32_t word = need_bits[warp];
    if (word == 0) { if (lane == 0) occ_bits[warp] = 0; return; }
    uint32_t view = (uint32_t)(warp / vwords);
    uint32_t rank = (uint32_t)(warp % vwords) * 32 + lane;
    bool occ = false;
    if ((word >> lane) & 1u) {
        const uint32_t v = vorder[rank];
        const ViewDev &V = views[view];
        float ox = verts[3 * (size_t)v], oy = verts[3 * (size_t)v + 1], oz = verts[3 * (size_t)v + 2];
        float dx = V.pos[0] - ox, dy = V.pos[1] - oy, dz = V.pos[2] - oz;   // :203
        float tmax = sqrtf(((0.0f + dx * dx) + dy * dy) + dz * dz);        // :204
        float tmin = tmax * 0.0001f;                                       // :205
        dx = dx / tmax; dy = dy / tmax; dz = dz / tmax;                    // :206
        occ = bvh_occluded(nodes, tri, num_tris, ox, oy, oz, dx, dy, dz, tmin, tmax, stack_overflow);
    }
    uint32_t res = __ballot_sync(0xffffffffu, occ);
    if (lane == 0) {
        occ_bits[warp] = res;
        atomicAdd(ray_count, (unsigned long long)__popc(word));
    }
    (void)Vn;
}

struct Tri2 { float v1x, v1y, v2x, v2y, v3x, v3y, detT, min_x, min_y, max_x, max_y; };

// tri.h:58-76
__device__ __forceinline__ bool tri_inside(const Tri2 &t, float x, float y)
{
    float dx = x - t.v3x, dy = y - t.v3y;
    float alpha = ((t.v2y - t.v3y) * dx + (t.v3x - t.v2x) * dy) / t.detT;
    if (alpha < 0.0f || alpha > 1.0f) return false;
    float beta = ((t.v3y - t.v1y) * dx + (t.v1x - t.v3x) * dy) / t.detT;
    if (beta < 0.0f || beta > 1.0f) return false;
    if (alpha + beta > 1.0f) return false;
    return true;
}

// mve::Image<uint8_t>::linear_at (u8 rounding) on the gradient image
__device__ __forceinline__ uint8_t linear_at_u8(const uint8_t *__restrict__ img, int w, int h, float x, float y)
{
    x = fmaxf(0.0f, fminf((float)(w - 1), x));
    y = fmaxf(0.0f, fminf((float)(h - 1), y));
    int fx = (int)x, fy = (int)y;
    int fx1 = min(fx + 1, w - 1), fy1 = min(fy + 1, h - 1);
    float w1 = x - (float)fx, w0 = 1.0f - w1;
    float w3 = y - (float)fy, w2 = 1.0f - w3;
    float r = (float)img[fx + (size_t)fy * w] * (w0 * w2) + (float)img[fx1 + (size_t)fy * w] * (w1 * w2)
        + (float)img[fx + (size_t)fy1 * w] * (w0 * w3) + (float)img[fx1 + (size_t)fy1 * w] * (w1 * w3) + 0.5f;
    return (uint8_t)r;
}

// texture_view.cpp:134-251 for outlier_removal == NONE
// mean_color != nullptr <=> outlier removal on: colours are sampled even for DATA_TERM_AREA (:159)
__device__ float face_quality(const ViewDev &V, Px p1, Px p2, Px p3, int data_term, float *mean_color)
{
    Tri2 t;
    t.v1x = p1.x; t.v1y = p1.y; t.v2x = p2.x; t.v2y = p2.y; t.v3x = p3.x; t.v3y = p3.y;
    {
        float T0 = p1.x - p3.x, T1 = p2.x - p3.x, T2 = p1.y - p3.y, T3 = p2.y - p3.y;
        t.detT = T0 * T3 - T2 * T1;
    }
    t.min_x = fminf(p1.x, fminf(p2.x, p3.x)); t.min_y = fminf(p1.y, fminf(p2.y, p3.y));
    t.max_x = fmaxf(p1.x, fmaxf(p2.x, p3.x)); t.max_y = fmaxf(p1.y, fmaxf(p2.y, p3.y));
    float area;
    {
        float u0 = p2.x - p1.x, u1 = p2.y - p1.y, v0 = p3.x - p1.x, v1 = p3.y - p1.y;
        area = 0.5f * fabsf(u0 * v1 - u1 * v0);
    }
    if (area < 1.1920928955078125e-07f) return 0.0f;  // FLT_EPSILON :150
    if (data_term != 1 && !mean_color) return area;   // DATA_TERM_AREA, no sampling (:159,:248)

    unsigned long long num_samples = 0;
    double gmi = 0.0;
    double colors[3] = {0.0, 0.0, 0.0};
    const uint8_t *__restrict__ grad = V.grad;
    const int w = V.w;
    if (area > 0.5f) {
        for (;;) {  // :163-167
            if (p1.y <= p2.y) {
                if (p2.y <= p3.y) break;
                Px tmp = p2; p2 = p3; p3 = tmp;
            } else {
                Px tmp = p1; p1 = p2; p2 = tmp;
            }
        }
        const float m1 = (p1.y - p3.y) / (p1.x - p3.x);
        const float b1 = p1.y - m1 * p1.x;
        const float m2 = (p1.y - p2.y) / (p1.x - p2.x);
        const float b2 = p1.y - m2 * p1.x;
        const float m3 = (p2.y - p3.y) / (p2.x - p3.x);
        const float b3 = p2.y - m3 * p2.x;
        const bool fast = isfinite(m1) && m2 != 0.0f && isfinite(m2) && m3 != 0.0f && isfinite(m3);
        const int y0 = (int)floorf(t.min_y);
        const float y_end = ceilf(t.max_y);
        for (int y = y0; (float)y < y_end; ++y) {
            float min_x = t.min_x - 0.5f;
            float max_x = t.max_x + 0.5f;
            if (fast) {
                const float cy = (float)y + 0.5f;
                min_x = (cy - b1) / m1;
                if (cy <= p2.y) max_x = (cy - b2) / m2;
                else max_x = (cy - b3) / m3;
                if (min_x >= max_x) { float s = min_x; min_x = max_x; max_x = s; }
                if (min_x < t.min_x || min_x > t.max_x) continue;
                if (max_x < t.min_x || max_x > t.max_x) continue;
            }
            const int x0 = (int)floorf(min_x + 0.5f);
            const float x_end = ceilf(max_x - 0.5f);
            for (int x = x0; (float)x < x_end; ++x) {
                const float cx = (float)x + 0.5f;
                const float cy = (float)y + 0.5f;
                if (!fast && !tri_inside(t, cx, cy)) continue;
                if (mean_color) {  // :207-212
                    const uint8_t *px = V.rgb + 3 * ((size_t)x + (size_t)y * w);
                    colors[0] += (double)px[0] / 255.0; colors[1] += (double)px[1] / 255.0; colors[2] += (double)px[2] / 255.0;
                }
                if (data_term == 1) gmi += (double)grad[(size_t)x + (size_t)y * w] / 255.0;
                ++num_samples;
            }
        }
    }
    if (mean_color) {  // :233-245
        if (num_samples > 0) {
            for (int i = 0; i < 3; ++i) mean_color[i] = (float)(colors[i] / (double)num_samples);
        } else {
            for (int i = 0; i < 3; ++i) {
                double c1 = (double)linear_at_rgb(V.rgb, V.w, V.h, p1.x, p1.y, i) / 255.0;
                double c2 = (double)linear_at_rgb(V.rgb, V.w, V.h, p2.x, p2.y, i) / 255.0;
                double c3 = (double)linear_at_rgb(V.rgb, V.w, V.h, p3.x, p3.y, i) / 255.0;
                mean_color[i] = (float)((c1 + c2 + c3) / 3.0);
            }
        }
    }
    if (data_term != 1) return area;
    if (num_samples > 0) {
        gmi = (gmi / (double)num_samples) * (double)area;
    } else {
        double g1 = (double)linear_at_u8(grad, V.w, V.h, p1.x, p1.y) / 255.0;
        double g2 = (double)linear_at_u8(grad, V.w, V.h, p2.x, p2.y) / 255.0;
        double g3 = (double)linear_at_u8(grad, V.w, V.h, p3.x, p3.y) / 255.0;
        gmi = ((g1 + g2 + g3) / 3.0) * (double)area;
    }
    return (float)gmi;
}

__global__ void __launch_bounds__(256) k_quality(const float *__restrict__ verts, const uint32_t *__restrict__ faces,
                                                 const ViewDev *__restrict__ views,
                                                 const uint16_t *__restrict__ cand_view,
                                                 const uint32_t *__restrict__ cand_face, uint64_t num_cand,
                                                 const uint32_t *__restrict__ occ_bits, uint32_t vwords,
                                                 const uint32_t *__restrict__ vrank,
                                                 int data_term, float *cand_q, uint32_t *max_q_bits,
                                                 float *cand_ycc /* [ncand][3] or null */)
{
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    float q = 0.0f;
    if (i < num_cand) {
        uint32_t f = cand_face[i];
        uint32_t j = cand_view[i];
        FaceGeom g;
        uint32_t vid[3];
        load_face(verts, faces, nullptr, f, g, vid);
        bool visible = true;
        if (occ_bits) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const uint32_t r = vrank[vid[k]];
                if ((occ_bits[(size_t)j * vwords + (r >> 5)] >> (r & 31)) & 1u) visible = false;
            }
        }
        if (visible) {
            const ViewDev &V = views[j];
            Px p1 = pixel_coords(V, g.v[0]), p2 = pixel_coords(V, g.v[1]), p3 = pixel_coords(V, g.v[2]);
            float mc[3] = {0.0f, 0.0f, 0.0f};
            q = face_quality(V, p1, p2, p3, data_term, cand_ycc ? mc : nullptr);
            if (cand_ycc) {  // mve::image::color_rgb_to_ycbcr<float> (:225)
                cand_ycc[3 * i + 0] = (mc[0] * 0.299f + mc[1] * 0.587f) + mc[2] * 0.114f;
                cand_ycc[3 * i + 1] = ((mc[0] * -0.168736f + mc[1] * -0.331264f) + mc[2] * 0.5f) + 0.5f;
                cand_ycc[3 * i + 2] = ((mc[0] * 0.5f + mc[1] * -0.418688f) + mc[2] * -0.081312f) + 0.5f;
            }
        }
        cand_q[i] = q;
    }
    // qualities are >= 0 (or NaN, which the reference's std::max also ignores): uint order == float order
    uint32_t qb = (q == q) ? __float_as_uint(q) : 0u;
    for (int s = 16; s; s >>= 1) qb = max(qb, __shfl_xor_sync(0xffffffffu, qb, s));
    if ((threadIdx.x & 31) == 0 && qb && !cand_ycc) atomicMax(max_q_bits, qb);  // with outlier removal the
}                                                                             // maximum is taken afterwards

// ---- photometric outlier detection (calculate_data_costs.cpp:35-129), one thread per face ------------
// Restates oracle/datacosts.c photometric_outlier_detection operation by operation (fp64, no FMA):
// sequential mean / covariance sums over the face's infos in ascending view order, FullPivLU<3x3>
// inverse (full pivoting, rank threshold eps*3*|max pivot|), exp((-0.5 d) Cinv d^T).
__device__ bool lu3_inverse(const double *A, double *inv)
{
    double lu[9];
    for (int i = 0; i < 9; ++i) lu[i] = A[i];
    int rt[3], ct[3];
    double maxpivot = 0.0;
    int nonzero = 3;
    for (int k = 0; k < 3; ++k) {
        int br = k, bc = k;
        double biggest = -1.0;
        for (int cc = k; cc < 3; ++cc)
            for (int rr = k; rr < 3; ++rr) {
                double a = fabs(lu[rr * 3 + cc]);
                if (a > biggest) { biggest = a; br = rr; bc = cc; }
            }
        if (biggest == 0.0) { nonzero = k; for (int i = k; i < 3; ++i) { rt[i] = i; ct[i] = i; } break; }
        if (biggest > maxpivot) maxpivot = biggest;
        rt[k] = br; ct[k] = bc;
        if (br != k) for (int cc = 0; cc < 3; ++cc) { double t = lu[k * 3 + cc]; lu[k * 3 + cc] = lu[br * 3 + cc]; lu[br * 3 + cc] = t; }
        if (bc != k) for (int rr = 0; rr < 3; ++rr) { double t = lu[rr * 3 + k]; lu[rr * 3 + k] = lu[rr * 3 + bc]; lu[rr * 3 + bc] = t; }
        for (int rr = k + 1; rr < 3; ++rr) lu[rr * 3 + k] = lu[rr * 3 + k] / lu[k * 3 + k];
        for (int rr = k + 1; rr < 3; ++rr)
            for (int cc = k + 1; cc < 3; ++cc) lu[rr * 3 + cc] = lu[rr * 3 + cc] - lu[rr * 3 + k] * lu[k * 3 + cc];
    }
    int rank = 0;
    const double thr = maxpivot * (2.220446049250313e-16 * 3.0);
    for (int i = 0; i < nonzero; ++i) if (fabs(lu[i * 3 + i]) > thr) ++rank;
    if (rank != 3) return false;
    for (int col = 0; col < 3; ++col) {
        double c[3] = {0.0, 0.0, 0.0};
        c[col] = 1.0;
        for (int k = 0; k < 3; ++k) if (rt[k] != k) { double t = c[k]; c[k] = c[rt[k]]; c[rt[k]] = t; }
        for (int i = 1; i < 3; ++i) for (int j = 0; j < i; ++j) c[i] = c[i] - lu[i * 3 + j] * c[j];
        for (int i = 2; i >= 0; --i) {
            for (int j = i + 1; j < 3; ++j) c[i] = c[i] - lu[i * 3 + j] * c[j];
            c[i] = c[i] / lu[i * 3 + i];
        }
        for (int k = 2; k >= 0; --k) if (ct[k] != k) { double t = c[k]; c[k] = c[ct[k]]; c[ct[k]] = t; }
        for (int i = 0; i < 3; ++i) inv[i * 3 + col] = c[i];
    }
    return true;
}

__device__ __forceinline__ double gauss3(const float *x, const double *mu, const double *ci)
{
    double d[3], t[3], r[3];
    for (int i = 0; i < 3; ++i) { d[i] = (double)x[i] - mu[i]; t[i] = -0.5 * d[i]; }
    for (int j = 0; j < 3; ++j) r[j] = (t[0] * ci[0 * 3 + j] + t[1] * ci[1 * 3 + j]) + t[2] * ci[2 * 3 + j];
    return exp((r[0] * d[0] + r[1] * d[1]) + r[2] * d[2]);
}

__global__ void __launch_bounds__(128) k_outlier(const uint64_t *__restrict__ cand_ptr, float *cand_q,
                                                 const float *__restrict__ cand_ycc, uint8_t *flag,
                                                 uint32_t face_begin, uint32_t face_end, int mode,
                                                 uint32_t *max_q_bits)
{
    const uint32_t f = face_begin + blockIdx.x * blockDim.x + threadIdx.x;
    float qmax = 0.0f;
    if (f < face_end) {
        const uint64_t a = cand_ptr[f], b = cand_ptr[f + 1];
        // infos of this face = candidates with quality != 0 (:222), ascending view order
        uint32_t n = 0;
        for (uint64_t i = a; i < b; ++i) { const bool in = cand_q[i] != 0.0f; flag[i] = in ? 1 : 2; n += in; }  // 2 = not an info
        const double gauss_rejection_threshold = 6e-3, minimal_covariance = 5e-4;
        const double factor = mode == 2 ? 1.0 : (double)0.2f;
        bool done = n == 0;
        uint32_t rows = n;
        double mean[3], cov[9], cinv[9];
        for (int it = 0; it < 10 && !done; ++it) {
            if (rows < 4u) { done = true; break; }
            for (int i = 0; i < 3; ++i) mean[i] = 0.0;
            for (uint64_t i = a; i < b; ++i) if (flag[i] == 1) for (int k = 0; k < 3; ++k) mean[k] += (double)cand_ycc[3 * i + k];
            for (int i = 0; i < 3; ++i) mean[i] = mean[i] / (double)rows;
            for (int i = 0; i < 9; ++i) cov[i] = 0.0;
            for (uint64_t i = a; i < b; ++i) if (flag[i] == 1) {
                double c[3];
                for (int k = 0; k < 3; ++k) c[k] = (double)cand_ycc[3 * i + k] - mean[k];
                for (int k = 0; k < 3; ++k) for (int j = 0; j < 3; ++j) cov[k * 3 + j] += c[k] * c[j];
            }
            double maxabs = 0.0;
            for (int i = 0; i < 9; ++i) { cov[i] = cov[i] / (double)(rows - 1); if (fabs(cov[i]) > maxabs) maxabs = fabs(cov[i]); }
            if (maxabs < minimal_covariance) {
                for (uint64_t i = a; i < b; ++i) if (flag[i] == 0) cand_q[i] = 0.0f;
                done = true;
                break;
            }
            if (!lu3_inverse(cov, cinv)) { done = true; break; }
            rows = 0;
            for (uint64_t i = a; i < b; ++i) if (flag[i] != 2) {
                const uint8_t in = gauss3(cand_ycc + 3 * i, mean, cinv) >= gauss_rejection_threshold ? 1 : 0;
                flag[i] = in;
                rows += in;
            }
        }
        if (!done) {
            for (int i = 0; i < 9; ++i) cinv[i] = cinv[i] * factor;
            for (uint64_t i = a; i < b; ++i) if (flag[i] != 2) {
                const double g = gauss3(cand_ycc + 3 * i, mean, cinv);
                if (mode == 1) cand_q[i] = (float)((double)cand_q[i] * g);
                else if (g < gauss_rejection_threshold) cand_q[i] = 0.0f;
            }
        }
        for (uint64_t i = a; i < b; ++i) { const float q = cand_q[i]; if (q == q) qmax = fmaxf(qmax, q); }
    }
    uint32_t qb = __float_as_uint(qmax);
    for (int s = 16; s; s >>= 1) qb = max(qb, __shfl_xor_sync(0xffffffffu, qb, s));
    if ((threadIdx.x & 31) == 0 && qb) atomicMax(max_q_bits, qb);
}

__global__ void k_count_survivors(const uint64_t *__restrict__ cand_ptr, const float *__restrict__ cand_q,
                                  uint32_t face_begin, uint32_t face_end, uint32_t F, uint64_t *cnt)
{
    uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f > F) return;
    uint64_t n = 0;
    if (f >= face_begin && f < face_end)
        for (uint64_t i = cand_ptr[f]; i < cand_ptr[f + 1]; ++i) n += (cand_q[i] != 0.0f);  // :222
    cnt[f] = n;
}

// drop quality 0, warp per face in 32-candidate chunks: bit k of `m` = candidate c+k survives, so a kept candidate's slot
// is the face's offset + the survivors of the earlier chunks + popc(m & lanemask_lt), and the DataCosts rows are written
// in contiguous runs in candidate (= ascending view) order
__global__ void __launch_bounds__(256) k_compact(const uint64_t *__restrict__ cand_ptr, const float *__restrict__ cand_q,
                                                 const uint16_t *__restrict__ cand_view, const uint64_t *__restrict__ dc_ptr,
                                                 uint32_t face_begin, uint32_t face_end, uint16_t *dc_view, float *dc_quality)
{
    const uint32_t lane = threadIdx.x & 31u, lt = lanemask_lt();
    for (uint32_t f = face_begin + warp_id(); f < face_end; f += num_warps()) {
        const uint64_t a = cand_ptr[f], b = cand_ptr[f + 1];
        uint64_t o = dc_ptr[f];
        for (uint64_t c = a; c < b; c += 32) {
            const uint32_t n = b - c < 32 ? (uint32_t)(b - c) : 32u;
            uint32_t m = 0;
            for (uint32_t k = 0; k < n; ++k) m |= (uint32_t)(cand_q[c + k] != 0.0f) << k;   // broadcast loads of one chunk
            if ((m >> lane) & 1u) {
                const uint64_t slot = o + __popc(m & lt);
                dc_view[slot] = cand_view[c + lane];
                dc_quality[slot] = cand_q[c + lane];
            }
            o += __popc(m);
        }
    }
}

constexpr int HIST_BINS = 10000;

// histogram.cpp:27-34 with min = 0
__global__ void __launch_bounds__(512) k_histogram(const float *__restrict__ q, uint64_t n, float vmax,
                                                   uint32_t *bins)
{
    __shared__ uint32_t sb[HIST_BINS];
    for (int i = threadIdx.x; i < HIST_BINS; i += blockDim.x) sb[i] = 0;
    __syncthreads();
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        float c = fmaxf(0.0f, fminf(vmax, q[i]));
        uint32_t idx = (uint32_t)floorf(((c - 0.0f) / (vmax - 0.0f)) * (float)(HIST_BINS - 1));
        atomicAdd(&sb[idx], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < HIST_BINS; i += blockDim.x)
        if (sb[i]) atomicAdd(&bins[i], sb[i]);
}

// calculate_data_costs.cpp:295-296
__global__ void k_normalize(const float *__restrict__ q, uint64_t n, float percentile, float *cost)
{
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float normalized = fminf(1.0f, q[i] / percentile);
    cost[i] = 1.0f - normalized;
}

// smallest float c with !(double(acosf(c)) > MATH_DEG2RAD(75.0f)); acosf is the host libm's, as in
// the reference build.  The device then rejects viewing_angle < c (calculate_data_costs.cpp:187).
float cos75_threshold()
{
    const double thr = 75.0f * (3.14159265358979323846264338327950288 / 180.0);
    uint32_t lo = 0;  // 0.0f: acos = pi/2 > thr (rejected)
    float one = 1.0f;
    uint32_t hi;
    memcpy(&hi, &one, 4);  // acos(1) = 0 (kept)
    while (hi - lo > 1) {
        uint32_t mid = lo + (hi - lo) / 2;
        float m;
        memcpy(&m, &mid, 4);
        if ((double)acosf(m) > thr) lo = mid; else hi = mid;
    }
    float r;
    memcpy(&r, &hi, 4);
    return r;
}

}  // namespace

// grid of the warp-per-face kernels (256 threads = 8 warps per block): one warp per face up to a full-occupancy wave,
// beyond that the warps loop over the faces
static unsigned face_warp_blocks(const b2tex_ctx *c, uint64_t faces)
{
    const uint64_t want = (faces + 7) / 8;
    const uint64_t wave = (uint64_t)std::max(1, c->num_sms) * 8;
    return (unsigned)std::max<uint64_t>(1, std::min(want, wave));
}

// qualities of all candidates are known: photometric outlier removal (optional), drop quality 0, compact to the
// DataCosts layout, maximum (calculate_data_costs.cpp:222,265-281)
static int finish_candidates(b2tex_ctx *c, const b2tex_settings *st, uint64_t num_cand, b2tex_dc_info *info)
{
    cudaStream_t s = c->stream;
    const uint32_t F = c->F, fb = c->face_begin, fe = c->face_end, nf = fe - fb;
    const bool outlier = st->outlier_removal != 0;
    DevBuf<uint64_t> &cnt = c->s_cnt64;
    unsigned long long *ray_count = reinterpret_cast<unsigned long long *>(c->scalars.p + 2);
    if (outlier && nf) {
        ScopedTimer tm(c, "k_outlier", 16.0 * (double)num_cand);
        B2_LAUNCH k_outlier<<<(nf + 127) / 128, 128, 0, s>>>(c->cand_ptr.p, c->cand_q.p, c->cand_ycc.p, c->cand_flag.p, fb, fe,
                                                   st->outlier_removal, c->scalars.p);
        B2_KERNEL_CHECK();
    }
    {
        ScopedTimer tm(c, "k_count_survivors", 4.0 * (double)num_cand + 16.0 * F);
        B2_LAUNCH k_count_survivors<<<(F + 1 + 255) / 256, 256, 0, s>>>(c->cand_ptr.p, c->cand_q.p, fb, fe, F, cnt.p);
    }
    B2_KERNEL_CHECK();
    B2_TRY(cub_exclusive_sum_u64(c, cnt.p, c->dc_ptr.p, (size_t)F + 1));
    uint64_t nnz = 0;
    uint32_t maxbits = 0;
    unsigned long long rays = 0;
    B2_CUDA(cudaMemcpyAsync(&nnz, c->dc_ptr.p + F, sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaMemcpyAsync(&maxbits, c->scalars.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaMemcpyAsync(&rays, ray_count, sizeof(rays), cudaMemcpyDeviceToHost, s));
    uint32_t stack_overflow = 0;
    B2_CUDA(cudaMemcpyAsync(&stack_overflow, c->scalars.p + 8, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaStreamSynchronize(s));
    if (stack_overflow) {   // the reference's BVH has no such limit: refuse rather than risk a face counted as visible
        set_error("visibility rays: the traversal stack (100 entries) overflowed");
        return B2TEX_ERR_LIMITS;
    }
    c->nnz = nnz;
    B2_TRY(c->dc_view.alloc(nnz));
    B2_TRY(c->dc_quality.alloc(nnz));
    B2_TRY(c->dc_cost.alloc(nnz));
    if (nf) {
        ScopedTimer tm(c, "k_compact", 6.0 * (double)num_cand + 6.0 * (double)nnz + 16.0 * nf);
        B2_LAUNCH k_compact<<<face_warp_blocks(c, nf), 256, 0, s>>>(c->cand_ptr.p, c->cand_q.p, c->cand_view.p, c->dc_ptr.p, fb, fe,
                                         c->dc_view.p, c->dc_quality.p);
    }
    B2_KERNEL_CHECK();
    float maxq;
    memcpy(&maxq, &maxbits, 4);
    info->nnz = nnz;
    info->candidates = num_cand;
    info->rays = rays;
    info->max_quality = maxq;
    info->percentile = 0.0f;
    return B2TEX_OK;
}

int data_costs_qualities(b2tex_ctx *c, const b2tex_settings *st, b2tex_dc_info *info)
{
    invalidate(c, COSTS);
    if (!c->F || !c->K) { set_error("data costs: mesh and views must be set first"); return B2TEX_ERR_ARG; }
    B2_TRY(require(c, MESH | PIXELS, "data costs"));
    if (st->outlier_removal < 0 || st->outlier_removal > 2) { set_error("unknown outlier removal mode"); return B2TEX_ERR_UNSUPPORTED; }
    const bool outlier = st->outlier_removal != 0;
    if (c->K > 65535u) { set_error("Exeeded maximal number of views"); return B2TEX_ERR_LIMITS; }
    cudaStream_t s = c->stream;
    // image preparation and the BVH are part of the stage in the reference
    // (calculate_data_costs.cpp:144,157-163), so they are redone on every call
    // The camera block first: BVH, culling and the visibility rays need no pixel, so with a deferred image upload
    // (one-shot entry points) they run while the images are still on their way; the pixel work (Sobel, validity masks)
    // follows right before k_quality, its first consumer.
    // (Views with a validity mask -- a zero-sum corner pixel -- are the exception: the cull reads the mask, so there the pixel
    // work comes first, as in the reference.)
    if (c->any_corner_flag) B2_TRY(prepare_images(c, st->data_term, true));
    else B2_TRY(prepare_views(c, st->data_term));
    const bool vis = st->geometric_visibility_test != 0;
    if (vis) B2_TRY(build_bvh(c, true));

    const uint32_t F = c->F, K = c->K, fb = c->face_begin, fe = c->face_end;
    const uint32_t nf = fe - fb;
    const uint32_t vwords = (c->Vn + 31) / 32;
    const uint32_t kwords = (c->K + 31) / 32;
    B2_TRY(c->s_pass_bits.alloc((size_t)(c->face_end - c->face_begin) * kwords));
    static const float cos_thr = cos75_threshold();

    B2_TRY(c->cand_ptr.alloc((size_t)F + 1));
    B2_TRY(c->dc_ptr.alloc((size_t)F + 1));
    DevBuf<uint64_t> &cnt = c->s_cnt64;
    B2_TRY(cnt.alloc((size_t)F + 1));
    B2_TRY(cnt.zero(s));
    B2_TRY(c->scalars.alloc(std::max<size_t>(c->scalars.n, 256)));
    B2_CUDA(cudaMemsetAsync(c->scalars.p, 0, 64 * sizeof(uint32_t), s));
    const uint32_t blocks = (nf + 255) / 256;
    const double mesh_bytes = 24.0 * nf + 12.0 * c->Vn;
    if (nf) {
        ScopedTimer tm(c, "k_cull<count>", mesh_bytes + 8.0 * nf);
        B2_LAUNCH k_cull<false><<<blocks, 256, 0, s>>>(c->verts.p, c->faces.p, c->normals.p, c->views_dev.p, K, fb, fe,
                                             cos_thr, cnt.p, nullptr, nullptr, nullptr, nullptr, vwords, nullptr, c->s_pass_bits.p, kwords);
    }
    B2_KERNEL_CHECK();
    B2_TRY(cub_exclusive_sum_u64(c, cnt.p, c->cand_ptr.p, (size_t)F + 1));
    uint64_t num_cand = 0;
    B2_CUDA(cudaMemcpyAsync(&num_cand, c->cand_ptr.p + F, sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaStreamSynchronize(s));
    c->num_cand = num_cand;
    B2_TRY(c->cand_view.alloc(num_cand));
    B2_TRY(c->cand_face.alloc(num_cand));
    B2_TRY(c->cand_q.alloc(num_cand));
    if (outlier) { B2_TRY(c->cand_ycc.alloc(3 * num_cand)); B2_TRY(c->cand_flag.alloc(num_cand)); }
    if (vis) {
        B2_TRY(c->need_bits.alloc((size_t)K * vwords));
        B2_TRY(c->occ_bits.alloc((size_t)K * vwords));
        B2_TRY(c->need_bits.zero(s));
    }
    if (nf) {
        // pass words + offsets read, candidates written; with the ray bitmaps also the face's vertex ranks
        ScopedTimer tm(c, "k_cull<fill>", (4.0 * kwords + 8.0 + (vis ? 24.0 : 0.0)) * nf + 6.0 * (double)num_cand);
        B2_LAUNCH k_cull<true><<<face_warp_blocks(c, nf), 256, 0, s>>>(c->verts.p, c->faces.p, c->normals.p, c->views_dev.p, K, fb, fe,
                                                                        cos_thr, nullptr, c->cand_ptr.p, c->cand_view.p, c->cand_face.p,
                                                                        vis ? c->need_bits.p : nullptr, vwords, c->vrank.p,
                                                                        c->s_pass_bits.p, kwords);
    }
    B2_KERNEL_CHECK();
    unsigned long long *ray_count = reinterpret_cast<unsigned long long *>(c->scalars.p + 2);
    if (vis) {
        size_t warps = (size_t)K * vwords;
        size_t rblocks = (warps * 32 + 255) / 256;
        ScopedTimer tm(c, "k_rays", 8.0 * (double)warps + 12.0 * c->Vn);
        B2_LAUNCH k_rays<<<(unsigned)rblocks, 256, 0, s>>>(c->verts.p, c->Vn, c->views_dev.p, K, c->need_bits.p, c->occ_bits.p,
                                                 vwords, c->vorder.p, c->bvh.nodes.p, c->bvh.tri.p, c->bvh.num_tris,
                                                 ray_count, c->scalars.p + 8);
        B2_KERNEL_CHECK();
    }
    if (!c->any_corner_flag) B2_TRY(prepare_images(c, st->data_term, true));   // waits for the upload if it is still in flight
    if (num_cand) {
        size_t qblocks = (num_cand + 255) / 256;
        ScopedTimer tm(c, "k_quality", 10.0 * (double)num_cand + mesh_bytes);
        B2_LAUNCH k_quality<<<(unsigned)qblocks, 256, 0, s>>>(c->verts.p, c->faces.p, c->views_dev.p, c->cand_view.p,
                                                    c->cand_face.p, num_cand, vis ? c->occ_bits.p : nullptr, vwords,
                                                    c->vrank.p,
                                                    st->data_term, c->cand_q.p, c->scalars.p,
                                                    outlier ? c->cand_ycc.p : nullptr);
        B2_KERNEL_CHECK();
    }
    return finish_candidates(c, st, num_cand, info);
}

// maximum of the uploaded qualities (without outlier removal nothing else computes it on this path)
__global__ void __launch_bounds__(256) k_max_quality(const float *__restrict__ q, uint64_t n, uint32_t *max_q_bits)
{
    uint32_t qb = 0;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const float v = q[i];
        if (v == v && v > 0.0f) qb = max(qb, __float_as_uint(v));
    }
    for (int s = 16; s; s >>= 1) qb = max(qb, __shfl_xor_sync(0xffffffffu, qb, s));
    if ((threadIdx.x & 31) == 0 && qb) atomicMax(max_q_bits, qb);
}

// tex::postprocess_face_infos (calculate_data_costs.cpp:253-306) on candidates the CALLER computed: per face the
// (view, quality[, mean YCbCr colour]) infos in ascending view order
int data_costs_postprocess(b2tex_ctx *c, const b2tex_settings *st, uint32_t F, const uint64_t *face_ptr, const uint16_t *view,
                           const float *quality, const float *mean_ycbcr, b2tex_dc_info *info)
{
    if (st->outlier_removal < 0 || st->outlier_removal > 2) { set_error("unknown outlier removal mode"); return B2TEX_ERR_UNSUPPORTED; }
    const bool outlier = st->outlier_removal != 0;
    if (outlier && !mean_ycbcr) { set_error("postprocess_face_infos: outlier removal needs the mean colours"); return B2TEX_ERR_ARG; }
    cudaStream_t s = c->stream;
    set_face_count(c, F);
    const uint64_t n = face_ptr[F];
    B2_TRY(c->cand_ptr.upload(face_ptr, (size_t)F + 1, s));
    B2_TRY(c->cand_view.upload(view, n, s));
    B2_TRY(c->cand_q.upload(quality, n, s));
    if (outlier) { B2_TRY(c->cand_ycc.upload(mean_ycbcr, 3 * n, s)); B2_TRY(c->cand_flag.alloc(n)); }
    B2_TRY(c->dc_ptr.alloc((size_t)F + 1));
    B2_TRY(c->s_cnt64.alloc((size_t)F + 1));
    B2_TRY(c->scalars.alloc(std::max<size_t>(c->scalars.n, 256)));
    B2_CUDA(cudaMemsetAsync(c->scalars.p, 0, 64 * sizeof(uint32_t), s));
    c->num_cand = n;
    if (!outlier && n) B2_LAUNCH k_max_quality<<<std::max(1, c->num_sms * 4), 256, 0, s>>>(c->cand_q.p, n, c->scalars.p);
    B2_KERNEL_CHECK();
    return finish_candidates(c, st, n, info);
}

int data_costs_histogram(b2tex_ctx *c, float gmax)
{
    cudaStream_t s = c->stream;
    B2_TRY(c->hist.alloc(HIST_BINS));
    B2_TRY(c->hist.zero(s));
    if (c->nnz) {
        int blocks = std::max(1, c->num_sms * 2);
        ScopedTimer tm(c, "k_histogram", 4.0 * (double)c->nnz);
        B2_LAUNCH k_histogram<<<blocks, 512, 0, s>>>(c->dc_quality.p, c->nnz, gmax, c->hist.p);
        B2_KERNEL_CHECK();
    }
    return B2TEX_OK;
}

int data_costs_normalize(b2tex_ctx *c, float gmax, const uint32_t *bins, b2tex_dc_info *info)
{
    // Histogram::get_approx_percentile(0.995f), histogram.cpp:49-63 (min = 0)
    long long num_values = 0;
    for (int i = 0; i < HIST_BINS; ++i) num_values += bins[i];
    long long num = 0;
    float upper_bound = 0.0f, percentile = gmax;
    for (int i = 0; i < HIST_BINS; ++i) {
        if ((float)num / (float)num_values > 0.995f) { percentile = upper_bound; break; }
        num += bins[i];
        upper_bound = ((float)i / (float)(HIST_BINS - 1)) * (gmax - 0.0f) + 0.0f;
    }
    if (c->nnz) {
        ScopedTimer tm(c, "k_normalize", 8.0 * (double)c->nnz);
        B2_LAUNCH k_normalize<<<(unsigned)((c->nnz + 255) / 256), 256, 0, c->stream>>>(c->dc_quality.p, c->nnz, percentile,
                                                                            c->dc_cost.p);
        B2_KERNEL_CHECK();
    }
    info->nnz = c->nnz;
    info->max_quality = gmax;
    info->percentile = percentile;
    mark_valid(c, COSTS);
    return B2TEX_OK;
}

}  // namespace b2
