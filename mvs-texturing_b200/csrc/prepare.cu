// prepare.cu -- tex::prepare_mesh (prepare_mesh.cpp:14-70) on the device: the redundant faces dropped, the face normals
// of the kept faces, the mesh graph of the kept faces (graph.cu) and angle-weighted vertex normals (DESIGN.md §4, "Mesh
// preparation").
//
//   validate : k_graph_validate (validate_faces, graph.cu): the lowest face with an index >= Vn
//   sets     : the distinct vertex set of every face, sorted and padded with its largest member: {a} -> (a,a,a),
//              {a,b} -> (a,b,b), {a,b,c} -> (a,b,c) for a < b < c.  (a,a,b), (b,a,a) and (a,b,b) share one set; a set has
//              fewer than 3 members exactly when s1 == s2.
//   sort     : (set, face) stably by set, faces ascending on input (CUB radix).  A set takes 3b bits, b = bits of Vn - 1:
//              one pass over the 64-bit key s0 << 2b | s1 << b | s2 when 3b <= 64, else two stable passes, by s1 << b | s2
//              and then by s0.  Either way every set becomes a run of ascending faces.
//   runs     : a face that is not the last of its run is redundant (a later face has the same set).  The last faces of the
//              runs of sets with fewer than 3 members form the table (set, largest face id), sorted by set.
//   subsets  : only when that table is not empty: a face is also redundant when a proper subset of its set (3 pairs and 3
//              singletons of a triangle, 2 singletons of a pair) is in the table with a larger face id.  Together: face i
//              goes when some face j > i has all its vertices among those of i (prepare_mesh.cpp:22-40), and no vertex
//              ring is scanned.
//   compact  : exclusive scan of the keep flags: the kept faces in their order, the input id of each, their face normals
//   graph    : build_mesh_graph on the kept faces, unchanged
//   vnormals : thread per vertex over its vf row: the faces ascending, which is MVE's face loop restricted to the vertex
// CUB only for the radix sorts and the scans.  Scratch: the grow-only buffers of the graph build (g_key, g_val, g_cnt).
#include <cub/cub.cuh>

#include "common.cuh"

namespace b2 {
namespace {

// the distinct vertex set of the face (a, b, c) as (s0, s1, s2), see the file comment
__device__ __forceinline__ void face_set(uint32_t a, uint32_t b, uint32_t c, uint32_t s[3])
{
    const uint32_t lo = min(a, b), hi = max(a, b);
    if (c < lo) { s[0] = c; s[1] = lo; s[2] = hi; }
    else if (c < hi) { s[0] = lo; s[1] = c; s[2] = hi; }
    else { s[0] = lo; s[1] = hi; s[2] = c; }
    if (s[0] == s[1]) s[1] = s[2];
}

// cross(b - a, c - a) of face (a, b, c) into n; returns its length (no FMA: -fmad=false)
__device__ __forceinline__ float face_cross(const float *verts, uint32_t a, uint32_t b, uint32_t c, float n[3])
{
    const float *A = verts + 3 * (size_t)a, *B = verts + 3 * (size_t)b, *C = verts + 3 * (size_t)c;
    const float u0 = B[0] - A[0], u1 = B[1] - A[1], u2 = B[2] - A[2];
    const float v0 = C[0] - A[0], v1 = C[1] - A[1], v2 = C[2] - A[2];
    n[0] = u1 * v2 - u2 * v1;
    n[1] = u2 * v0 - u0 * v2;
    n[2] = u0 * v1 - u1 * v0;
    return sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
}

// set[3f..3f+2] of every face; the first sort's key and the face ids
__global__ void k_prep_keys(const uint32_t *faces, uint32_t F, int bits, bool narrow, uint32_t *set, uint64_t *key,
                            uint32_t *ids)
{
    for (uint32_t f = blockIdx.x * blockDim.x + threadIdx.x; f < F; f += gridDim.x * blockDim.x) {
        uint32_t s[3];
        face_set(faces[3 * (size_t)f], faces[3 * (size_t)f + 1], faces[3 * (size_t)f + 2], s);
        set[3 * (size_t)f] = s[0]; set[3 * (size_t)f + 1] = s[1]; set[3 * (size_t)f + 2] = s[2];
        const uint64_t low = ((uint64_t)s[1] << bits) | s[2];
        key[f] = narrow ? ((uint64_t)s[0] << (2 * bits)) | low : low;
        ids[f] = f;
    }
}

// the second pass's key (wide sets): s0 of the face at every position of the first pass
__global__ void k_prep_first_member(const uint32_t *set, const uint32_t *ids, uint32_t F, uint32_t *key)
{
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < F; p += gridDim.x * blockDim.x) key[p] = set[3 * (size_t)ids[p]];
}

__device__ __forceinline__ bool same_set(const uint32_t *set, uint32_t f, uint32_t g)
{
    return set[3 * (size_t)f] == set[3 * (size_t)g] && set[3 * (size_t)f + 1] == set[3 * (size_t)g + 1] &&
           set[3 * (size_t)f + 2] == set[3 * (size_t)g + 2];
}

// keep[f] = f is the last face of its run; tail[p] = position p ends the run of a set with fewer than 3 members.
// p = F writes keep[F] = tail[F] = 0 (the scans' last entries).
__global__ void k_prep_runs(const uint32_t *set, const uint32_t *sorted, uint32_t F, uint32_t *keep, uint32_t *tail)
{
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p <= F; p += gridDim.x * blockDim.x) {
        if (p == F) { keep[F] = 0; tail[F] = 0; continue; }
        const uint32_t f = sorted[p];
        const bool last = p + 1 == F || !same_set(set, f, sorted[p + 1]);
        keep[f] = last;
        tail[p] = last && set[3 * (size_t)f + 1] == set[3 * (size_t)f + 2];
    }
}

// table[tpos[p]] = (set, face) of every flagged run tail: ascending by set
__global__ void k_prep_table(const uint32_t *set, const uint32_t *sorted, const uint32_t *tail, const uint32_t *tpos,
                             uint32_t F, uint4 *table)
{
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < F; p += gridDim.x * blockDim.x) {
        if (!tail[p]) continue;
        const uint32_t f = sorted[p];
        table[tpos[p]] = make_uint4(set[3 * (size_t)f], set[3 * (size_t)f + 1], set[3 * (size_t)f + 2], f);
    }
}

// the set (a, b, c) is in the table with a face id > f
__device__ __forceinline__ bool later_subset(const uint4 *table, uint32_t D, uint32_t a, uint32_t b, uint32_t c, uint32_t f)
{
    uint32_t lo = 0, hi = D;
    while (lo < hi) {
        const uint32_t m = lo + (hi - lo) / 2;
        const uint4 t = table[m];
        const bool less = t.x != a ? t.x < a : (t.y != b ? t.y < b : t.z < c);
        if (less) lo = m + 1; else hi = m;
    }
    return lo < D && table[lo].x == a && table[lo].y == b && table[lo].z == c && table[lo].w > f;
}

// a kept face with a proper subset of its set in the table at a larger face id is redundant too
__global__ void k_prep_subsets(const uint32_t *set, uint32_t F, const uint4 *table, uint32_t D, uint32_t *keep)
{
    for (uint32_t f = blockIdx.x * blockDim.x + threadIdx.x; f < F; f += gridDim.x * blockDim.x) {
        if (!keep[f]) continue;
        const uint32_t a = set[3 * (size_t)f], b = set[3 * (size_t)f + 1], c = set[3 * (size_t)f + 2];
        if (a == b) continue;   // a singleton: no proper subset
        bool red = later_subset(table, D, a, a, a, f) || later_subset(table, D, b, b, b, f);
        if (b != c)             // a triangle: its pairs and its third singleton
            red = red || later_subset(table, D, c, c, c, f) || later_subset(table, D, a, b, b, f) ||
                  later_subset(table, D, a, c, c, f) || later_subset(table, D, b, c, c, f);
        if (red) keep[f] = 0;
    }
}

// kept face f -> position kpos[f]: its indices, its input id and its normal; scal[1] counts the zero normals
__global__ void k_prep_compact(const uint32_t *faces, const float *verts, uint32_t F, const uint32_t *keep,
                               const uint32_t *kpos, uint32_t *out_faces, uint32_t *kept, float *normals,
                               unsigned long long *scal)
{
    for (uint32_t f = blockIdx.x * blockDim.x + threadIdx.x; f < F; f += gridDim.x * blockDim.x) {
        if (!keep[f]) continue;
        const size_t q = kpos[f];
        const uint32_t a = faces[3 * (size_t)f], b = faces[3 * (size_t)f + 1], c = faces[3 * (size_t)f + 2];
        out_faces[3 * q] = a; out_faces[3 * q + 1] = b; out_faces[3 * q + 2] = c;
        kept[q] = f;
        float n[3];
        const float l = face_cross(verts, a, b, c, n);
        const bool ok = l > 0.0f;
#pragma unroll
        for (int k = 0; k < 3; ++k) normals[3 * q + k] = ok ? n[k] / l : 0.0f;
        if (!ok) atomicAdd(&scal[1], 1ull);
    }
}

// Angle-weighted vertex normal of every vertex over its vf row (faces ascending).  A face whose cross product has length
// fnl != 0 adds (n / fnl) * acos(clamp(dot(e1 / |e1|, e2 / |e2|), -1, 1)) at its corner v (e1, e2: the edges from v to the
// face's next and next-but-one vertex); a face with fnl == 0, which includes every face with a repeated vertex, adds
// nothing.  The sum is then divided by its length where that is > 0, else the normal is 0.  oracle/prepare_mesh.c states
// the same operation order.
__global__ void k_prep_vertex_normals(const float *verts, const uint32_t *faces, const uint32_t *vf_ptr,
                                      const uint32_t *vf_idx, uint32_t nv, float *vn)
{
    for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += gridDim.x * blockDim.x) {
        float acc[3] = {0.0f, 0.0f, 0.0f};
        for (uint32_t r = vf_ptr[v]; r < vf_ptr[v + 1]; ++r) {
            const size_t f = vf_idx[r];
            const uint32_t a = faces[3 * f], b = faces[3 * f + 1], c = faces[3 * f + 2];
            float n[3];
            const float fnl = face_cross(verts, a, b, c, n);
            if (fnl == 0.0f) continue;
            // the corner at v: (p, q, r) = the face's vertices starting there, in the face's order
            const uint32_t p = a == v ? a : (b == v ? b : c), q = a == v ? b : (b == v ? c : a), r3 = a == v ? c : (b == v ? a : b);
            const float *P = verts + 3 * (size_t)p, *Q = verts + 3 * (size_t)q, *R = verts + 3 * (size_t)r3;
            float e1[3] = {Q[0] - P[0], Q[1] - P[1], Q[2] - P[2]}, e2[3] = {R[0] - P[0], R[1] - P[1], R[2] - P[2]};
            const float l1 = sqrtf(e1[0] * e1[0] + e1[1] * e1[1] + e1[2] * e1[2]);
            const float l2 = sqrtf(e2[0] * e2[0] + e2[1] * e2[1] + e2[2] * e2[2]);
#pragma unroll
            for (int k = 0; k < 3; ++k) { e1[k] = e1[k] / l1; e2[k] = e2[k] / l2; }
            float d = e1[0] * e2[0] + e1[1] * e2[1] + e1[2] * e2[2];
            d = d < -1.0f ? -1.0f : (d > 1.0f ? 1.0f : d);
            const float angle = acosf(d);
#pragma unroll
            for (int k = 0; k < 3; ++k) acc[k] = acc[k] + (n[k] / fnl) * angle;
        }
        const float len = sqrtf(acc[0] * acc[0] + acc[1] * acc[1] + acc[2] * acc[2]);
#pragma unroll
        for (int k = 0; k < 3; ++k) vn[3 * (size_t)v + k] = len > 0.0f ? acc[k] / len : 0.0f;
    }
}

}  // namespace

int prepare_mesh(b2tex_ctx *c, b2tex_mesh_prep_info *info)
{
    cudaStream_t s = c->stream;
    const uint32_t F = c->F, nv = c->Vn;
    if (6ull * F > 0x7FFFFFFFull) {
        set_error("prepare_mesh: %u faces exceed the sort's 32-bit item count (at most %u)", F, 0x7FFFFFFFu / 6);
        return B2TEX_ERR_LIMITS;
    }
    const int bits = nv <= 2 ? 1 : 32 - __builtin_clz(nv - 1);   // vertex ids < 2^bits
    const bool narrow = 3 * bits <= 64;
    auto grid_of = [&](size_t n) { return (unsigned)std::min<size_t>((n + 255) / 256 + 1, (size_t)c->num_sms * 16); };
    const unsigned grid = grid_of((size_t)F + 1);
    ScopedTimer total(c, "prep_mesh");   // the whole call, graph build and host round trips included

    B2_TRY(validate_faces(c, c->faces.p, F, nv, "prepare_mesh", "prep_validate"));

    // scratch, all within what the graph build of F faces takes:
    //   g_key[0]  u64 [F] first sort's keys; as u32: second pass keys [F] + sorted [F], run tails [F+1], their scan [F+1]
    //   g_key[1]  u64 [F] sorted keys, then the table uint4 [D <= F]
    //   g_val[0]  the sets [3F];  g_val[1]  the kept faces [3F']
    //   g_cnt     face ids [F] x 2, keep flags [F+1], their scan [F+1]
    B2_TRY(c->g_key[0].alloc(3 * (size_t)F));
    B2_TRY(c->g_key[1].alloc(2 * (size_t)F));
    B2_TRY(c->g_val[0].alloc(3 * (size_t)F));
    B2_TRY(c->g_val[1].alloc(3 * (size_t)F));
    B2_TRY(c->g_cnt.alloc(4 * (size_t)F + 2));
    uint32_t *set = c->g_val[0].p;
    uint32_t *k32 = (uint32_t *)c->g_key[0].p, *tail = k32 + 2 * (size_t)F, *tpos = k32 + 3 * (size_t)F + 1;
    uint32_t *ids0 = c->g_cnt.p, *ids1 = ids0 + F, *keep = ids0 + 2 * (size_t)F, *kpos = ids0 + 3 * (size_t)F + 1;
    uint4 *table = (uint4 *)c->g_key[1].p;
    const uint32_t *sorted = ids1;
    {
        const int b1 = narrow ? 3 * bits : 2 * bits;
        const double pass64 = 2.0 * (8 + 4) * F, pass32 = 2.0 * (4 + 4) * F;
        ScopedTimer t(c, "prep_sort", 12.0 * F + 24.0 * F + ((b1 + 7) / 8) * pass64 +
                                          (narrow ? 0.0 : 20.0 * F + ((bits + 7) / 8) * pass32));
        B2_LAUNCH k_prep_keys<<<grid, 256, 0, s>>>(c->faces.p, F, bits, narrow, set, c->g_key[0].p, ids0);
        B2_KERNEL_CHECK();
        size_t tb = 0;
        B2_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, c->g_key[0].p, c->g_key[1].p, ids0, ids1, (int)F, 0, b1, s));
        B2_TRY(c->cub_tmp.alloc(tb));
        B2_CUDA(cub::DeviceRadixSort::SortPairs(c->cub_tmp.p, tb, c->g_key[0].p, c->g_key[1].p, ids0, ids1, (int)F, 0, b1, s));
        if (!narrow) {   // stable second pass by s0: the first pass's keys are dead
            B2_LAUNCH k_prep_first_member<<<grid, 256, 0, s>>>(set, ids1, F, k32);
            B2_KERNEL_CHECK();
            B2_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, k32, k32 + F, ids1, ids0, (int)F, 0, bits, s));
            B2_TRY(c->cub_tmp.alloc(tb));
            B2_CUDA(cub::DeviceRadixSort::SortPairs(c->cub_tmp.p, tb, k32, k32 + F, ids1, ids0, (int)F, 0, bits, s));
            sorted = ids0;
        }
    }
    uint32_t D = 0;
    {
        ScopedTimer t(c, "prep_runs", 4.0 * F + 2 * 12.0 * F + 8.0 * F + 8.0 * F);
        B2_LAUNCH k_prep_runs<<<grid, 256, 0, s>>>(set, sorted, F, keep, tail);
        B2_KERNEL_CHECK();
        B2_TRY(cub_exclusive_sum_u32(c, tail, tpos, (size_t)F + 1));
    }
    B2_CUDA(cudaMemcpyAsync(&D, tpos + F, sizeof(D), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaStreamSynchronize(s));
    if (D) {   // some face has a repeated vertex: the subset lookups
        ScopedTimer t(c, "prep_subsets", 4.0 * F + 8.0 * F + 16.0 * D + 12.0 * F + 8.0 * F + 6 * 16.0 * F);
        B2_LAUNCH k_prep_table<<<grid, 256, 0, s>>>(set, sorted, tail, tpos, F, table);
        B2_KERNEL_CHECK();
        B2_LAUNCH k_prep_subsets<<<grid, 256, 0, s>>>(set, F, table, D, keep);
        B2_KERNEL_CHECK();
    }
    B2_TRY(c->kept_ids.alloc(F));   // trimmed to F' below
    B2_TRY(c->normals.alloc(3 * (size_t)F));
    {
        ScopedTimer t(c, "prep_compact", 8.0 * (F + 1) + 8.0 * F + 12.0 * F + (12.0 + 36 + 4 + 12) * F);
        B2_TRY(cub_exclusive_sum_u32(c, keep, kpos, (size_t)F + 1));
        B2_LAUNCH k_prep_compact<<<grid, 256, 0, s>>>(c->faces.p, c->verts.p, F, keep, kpos, c->g_val[1].p, c->kept_ids.p,
                                                     c->normals.p, c->g_scal.p);
        B2_KERNEL_CHECK();
    }
    uint32_t Fk = 0;
    unsigned long long sc[2];
    B2_CUDA(cudaMemcpyAsync(&Fk, kpos + F, sizeof(Fk), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaMemcpyAsync(sc, c->g_scal.p, sizeof(sc), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaMemcpyAsync(c->faces.p, c->g_val[1].p, 3 * sizeof(uint32_t) * Fk, cudaMemcpyDeviceToDevice, s));
    B2_CUDA(cudaStreamSynchronize(s));
    c->faces.n = 3 * (size_t)Fk; c->normals.n = 3 * (size_t)Fk; c->kept_ids.n = Fk;
    c->F = Fk; c->face_begin = 0; c->face_end = Fk;
    mark_valid(c, MESH);

    b2tex_graph_info gi;
    B2_TRY(build_mesh_graph(c, &gi));
    B2_TRY(c->vnormals.alloc(3 * (size_t)nv));
    {
        ScopedTimer t(c, "prep_vertex_normals", 8.0 * nv + (4.0 + 12 + 36) * 3 * Fk + 12.0 * nv);
        if (nv) B2_LAUNCH k_prep_vertex_normals<<<grid_of(nv), 256, 0, s>>>(c->verts.p, c->faces.p, c->vf_ptr.p, c->vf_idx.p,
                                                                             nv, c->vnormals.p);
        B2_KERNEL_CHECK();
    }
    B2_CUDA(cudaStreamSynchronize(s));
    mark_valid(c, PREP);
    if (info) {
        info->num_faces_in = F;
        info->num_faces = Fk;
        info->num_redundant = F - Fk;
        info->num_zero_normals = (uint32_t)sc[1];
        info->graph = gi;
    }
    return B2TEX_OK;
}

}  // namespace b2
