// graph.cu -- mesh topology on the device: the face adjacency (build_adjacency_graph.cpp:16-53) and the vertex rings
// (vertex -> faces, vertex -> vertices) from the resident mesh, element for element what scene.face_adjacency /
// scene.vertex_rings give on the host (DESIGN.md §4, "Mesh graph").
//
//   validate     : every face index < Vn (one flag: the lowest bad face), before anything is indexed by vertex id
//   edge keys    : 3F undirected keys (lo << b | hi) with value 3f+s, stable radix sort (CUB): the faces of one edge form
//                  a run, ascending by face, then by slot; inverse map (f, s) -> sorted position
//   adjacency    : thread per face, count pass -> exclusive scan -> fill pass.  A row is merged from the face's three
//                  runs: lower neighbours ascending (three-way merge), then higher ones by slot, ascending inside a slot,
//                  each face at its first position only (binary search in the runs of the earlier slots).  O(n log n) in
//                  the row length n, no per-row storage: fins and fans of any size take the same path.
//   vf           : 3F (vertex, face) pairs stably sorted by vertex (face-major input: faces ascending per vertex);
//                  vf_ptr by run detection
//   vv           : 6F directed keys (v << b | u) sorted, run heads scanned and compacted; vv_ptr by run detection
// CUB only for the radix sorts and the scans (DESIGN.md §4); everything else is here.
#include <cub/cub.cuh>

#include "common.cuh"

namespace b2 {
namespace {

constexpr uint32_t GRAPH_NONE = 0xFFFFFFFFu;

// scal[0] = lowest face with an index >= nv (GRAPH_NONE when all are valid)
__global__ void k_graph_validate(const uint32_t *faces, uint32_t F, uint32_t nv, unsigned long long *scal)
{
    for (uint32_t f = blockIdx.x * blockDim.x + threadIdx.x; f < F; f += gridDim.x * blockDim.x) {
        const size_t o = 3 * (size_t)f;
        if (faces[o] >= nv || faces[o + 1] >= nv || faces[o + 2] >= nv) atomicMin(&scal[0], (unsigned long long)f);
    }
}

// entry i = 3f+s: the undirected edge (v_s, v_{s+1 mod 3}) of face f
__global__ void k_graph_edge_keys(const uint32_t *faces, uint32_t n3, int bits, uint64_t *key, uint32_t *val)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n3; i += gridDim.x * blockDim.x) {
        const uint32_t f = i / 3, s = i - 3 * f;
        const uint32_t a = faces[i], b = faces[3 * (size_t)f + (s == 2 ? 0 : s + 1)];
        key[i] = ((uint64_t)min(a, b) << bits) | max(a, b);
        val[i] = i;
    }
}

// inv[3f+s] = sorted position of (f, s)
__global__ void k_graph_inverse(const uint32_t *val, uint32_t n3, uint32_t *inv)
{
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n3; p += gridDim.x * blockDim.x) inv[val[p]] = p;
}

// first position of the run [b, e) (ascending faces) whose face is >= g
__device__ __forceinline__ uint32_t run_lower_bound(const uint32_t *val, uint32_t b, uint32_t e, uint32_t g)
{
    while (b < e) {
        const uint32_t m = b + (e - b) / 2;
        if (val[m] / 3 < g) b = m + 1; else e = m;
    }
    return b;
}

// The adjacency row of face a, written to out (FILL) or only counted.  rb/re: the runs of a's three edges.
template <bool FILL>
__device__ uint32_t adjacency_row(uint32_t a, const uint32_t rb[3], const uint32_t re[3], const uint32_t *val, uint32_t *out)
{
    uint32_t n = 0;
    // neighbours below a, ascending: three-way merge of the runs' prefixes (a slot whose edge is another slot's too walks
    // the same run twice; the duplicates arrive next to each other)
    uint32_t cur[3] = {rb[0], rb[1], rb[2]};
    uint32_t last = GRAPH_NONE;
    for (;;) {
        uint32_t best = a;
        int bs = -1;
#pragma unroll
        for (int s = 0; s < 3; ++s)
            if (cur[s] < re[s]) {
                const uint32_t g = val[cur[s]] / 3;
                if (g < best) { best = g; bs = s; }
            }
        if (bs < 0) break;
        ++cur[bs];
        if (best != last) {
            if (FILL) out[n] = best;
            ++n;
            last = best;
        }
    }
    // neighbours above a: slot by slot, ascending inside a slot; a face already reached through an earlier slot keeps
    // its first position.  cur[s] is now the first entry of run s with a face >= a.
#pragma unroll
    for (int s = 0; s < 3; ++s) {
        uint32_t prev = a;
        for (uint32_t p = cur[s]; p < re[s]; ++p) {
            const uint32_t g = val[p] / 3;
            if (g == prev) continue;   // a itself, or a face that holds this edge twice
            prev = g;
            bool seen = false;
            for (int t = 0; t < s && !seen; ++t) {
                if (rb[t] == rb[s]) { seen = true; break; }   // the same edge as an earlier slot
                const uint32_t q = run_lower_bound(val, rb[t], re[t], g);
                seen = q < re[t] && val[q] / 3 == g;
            }
            if (seen) continue;
            if (FILL) out[n] = g;
            ++n;
        }
    }
    return n;
}

// the run of sorted keys that holds position p
__device__ __forceinline__ void key_run(const uint64_t *key, uint32_t n3, uint32_t p, uint32_t &b, uint32_t &e)
{
    const uint64_t k = key[p];
    b = p;
    while (b > 0 && key[b - 1] == k) --b;
    e = p + 1;
    while (e < n3 && key[e] == k) ++e;
}

// count pass: cnt[a] = row length (cnt[F] = 0 for the scan); scal[1] = longest row, scal[2] = edges shared by more than
// two faces (counted at the run head), scal[3] = sum over the rows of max(n - 3, 0) (overflow check of the u32 offsets)
__global__ void k_graph_adj_count(const uint64_t *key, const uint32_t *val, const uint32_t *inv, uint32_t F,
                                  uint32_t *cnt, unsigned long long *scal)
{
    const uint32_t n3 = 3 * F;
    for (uint32_t a = blockIdx.x * blockDim.x + threadIdx.x; a <= F; a += gridDim.x * blockDim.x) {
        if (a == F) { cnt[F] = 0; continue; }
        uint32_t rb[3], re[3];
#pragma unroll
        for (int s = 0; s < 3; ++s) {
            const uint32_t p = inv[3 * a + s];
            key_run(key, n3, p, rb[s], re[s]);
            if (p == rb[s]) {   // (a, s) heads its run: count the distinct faces of the edge
                uint32_t d = 0, prev = GRAPH_NONE;
                for (uint32_t q = rb[s]; q < re[s] && d <= 2; ++q) {
                    const uint32_t g = val[q] / 3;
                    if (g != prev) { ++d; prev = g; }
                }
                if (d > 2) atomicAdd(&scal[2], 1ull);
            }
        }
        const uint32_t n = adjacency_row<false>(a, rb, re, val, nullptr);
        cnt[a] = n;
        if (n > 3) atomicAdd(&scal[3], (unsigned long long)(n - 3));
        if (n > scal[1]) atomicMax(&scal[1], (unsigned long long)n);
    }
}

__global__ void k_graph_adj_fill(const uint64_t *key, const uint32_t *val, const uint32_t *inv, uint32_t F,
                                 const uint32_t *adj_ptr, uint32_t *adj_idx)
{
    const uint32_t n3 = 3 * F;
    for (uint32_t a = blockIdx.x * blockDim.x + threadIdx.x; a < F; a += gridDim.x * blockDim.x) {
        uint32_t rb[3], re[3];
#pragma unroll
        for (int s = 0; s < 3; ++s) key_run(key, n3, inv[3 * a + s], rb[s], re[s]);
        adjacency_row<true>(a, rb, re, val, adj_idx + adj_ptr[a]);
    }
}

// face id of every corner (the values of the vertex -> face sort)
__global__ void k_graph_corner_faces(uint32_t n3, uint32_t *fid)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n3; i += gridDim.x * blockDim.x) fid[i] = i / 3;
}

// ptr[v] = first position of vertex v in the ascending vertex list vs[0, n); ptr[v] = n past the last one.  Position p
// writes the entries (vs[p-1], vs[p]]; p = n writes the tail: every entry of ptr[0, nv] exactly once.
__global__ void k_graph_ring_ptr(const uint32_t *vs, uint32_t n, uint32_t nv, uint32_t *ptr)
{
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p <= n; p += gridDim.x * blockDim.x) {
        const uint64_t lo = p == 0 ? 0 : (uint64_t)vs[p - 1] + 1, hi = p == n ? nv : vs[p];
        for (uint64_t v = lo; v <= hi; ++v) ptr[v] = p;
    }
}

// entry i = 3f+s: the directed edges (v_s, v_{s+1}) at i and (v_{s+1}, v_s) at n3 + i
__global__ void k_graph_directed_keys(const uint32_t *faces, uint32_t n3, int bits, uint64_t *key)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n3; i += gridDim.x * blockDim.x) {
        const uint32_t f = i / 3, s = i - 3 * f;
        const uint64_t a = faces[i], b = faces[3 * (size_t)f + (s == 2 ? 0 : s + 1)];
        key[i] = (a << bits) | b;
        key[n3 + i] = (b << bits) | a;
    }
}

__global__ void k_graph_run_heads(const uint64_t *key, uint32_t n, uint32_t *head)
{
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x)
        head[p] = p == 0 || key[p] != key[p - 1];
}

// compaction of the distinct directed keys: vv_idx[pos[p]] = u of every run head p, vv_ptr by the run rule of
// k_graph_ring_ptr on the vertices v; p = n (the tail) also stores the number of distinct keys in scal[4]
__global__ void k_graph_vv_scatter(const uint64_t *key, const uint32_t *head, const uint32_t *pos, uint32_t n, int bits,
                                   uint32_t nv, uint32_t *vv_ptr, uint32_t *vv_idx, unsigned long long *scal)
{
    const uint64_t mask = (1ull << bits) - 1;
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p <= n; p += gridDim.x * blockDim.x) {
        if (p < n && !head[p]) continue;
        const uint32_t q = p < n ? pos[p] : pos[n - 1] + head[n - 1];
        if (p < n) vv_idx[q] = (uint32_t)(key[p] & mask);
        else scal[4] = q;
        const uint64_t lo = p == 0 ? 0 : (key[p - 1] >> bits) + 1, hi = p == n ? nv : key[p] >> bits;
        for (uint64_t v = lo; v <= hi; ++v) vv_ptr[v] = q;
    }
}

}  // namespace

int build_mesh_graph(b2tex_ctx *c, b2tex_graph_info *info)
{
    cudaStream_t s = c->stream;
    invalidate(c, ADJ | RINGS);   // a failed build leaves no graph behind
    B2_TRY(require(c, MESH, "build_mesh_graph"));
    const uint32_t F = c->F, nv = c->Vn;
    if (6ull * F > 0x7FFFFFFFull) {
        set_error("build_mesh_graph: %u faces exceed the sort's 32-bit item count (at most %u)", F, 0x7FFFFFFFu / 6);
        return B2TEX_ERR_LIMITS;
    }
    const uint32_t n3 = 3 * F, n6 = 6 * F;
    const int bits = nv <= 2 ? 1 : 32 - __builtin_clz(nv - 1);   // vertex ids < 2^bits
    auto grid_of = [&](size_t n) { return (unsigned)std::min<size_t>((n + 255) / 256 + 1, (size_t)c->num_sms * 16); };
    const unsigned grid = grid_of((size_t)F + 1);
    ScopedTimer total(c, "graph_build");   // the whole call, host round trips included

    B2_TRY(validate_faces(c, c->faces.p, F, nv, "build_mesh_graph", "graph_validate"));

    B2_TRY(c->adj_ptr.alloc((size_t)F + 1));
    B2_TRY(c->vf_ptr.alloc((size_t)nv + 1));
    B2_TRY(c->vv_ptr.alloc((size_t)nv + 1));
    if (F == 0) {
        B2_TRY(c->adj_idx.alloc(0)); B2_TRY(c->vf_idx.alloc(0)); B2_TRY(c->vv_idx.alloc(0));
        B2_TRY(c->adj_ptr.zero(s)); B2_TRY(c->vf_ptr.zero(s)); B2_TRY(c->vv_ptr.zero(s));
        B2_CUDA(cudaStreamSynchronize(s));
        mark_valid(c, ADJ | RINGS);
        if (info) *info = b2tex_graph_info{0, 0, 0, 0, 0};
        return B2TEX_OK;
    }
    B2_TRY(c->g_key[0].alloc(n6)); B2_TRY(c->g_key[1].alloc(n6));
    B2_TRY(c->g_val[0].alloc(n3)); B2_TRY(c->g_val[1].alloc(n3));
    B2_TRY(c->g_cnt.alloc(n6));
    const int ebits = 2 * bits;
    const double sort_pass_bytes = 2.0 * (8 + 4) * n3, vv_pass_bytes = 2.0 * 8 * n6;
    const int passes = (ebits + 7) / 8;

    // ---- face adjacency ----
    {
        ScopedTimer t(c, "graph_edge_sort", 12.0 * n3 + 12.0 * n3 + passes * sort_pass_bytes + 8.0 * n3);
        B2_LAUNCH k_graph_edge_keys<<<grid_of(n3), 256, 0, s>>>(c->faces.p, n3, bits, c->g_key[0].p, c->g_val[0].p);
        B2_KERNEL_CHECK();
        size_t tb = 0;
        B2_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, c->g_key[0].p, c->g_key[1].p, c->g_val[0].p, c->g_val[1].p,
                                                (int)n3, 0, ebits, s));
        B2_TRY(c->cub_tmp.alloc(tb));
        B2_CUDA(cub::DeviceRadixSort::SortPairs(c->cub_tmp.p, tb, c->g_key[0].p, c->g_key[1].p, c->g_val[0].p,
                                                c->g_val[1].p, (int)n3, 0, ebits, s));
        B2_LAUNCH k_graph_inverse<<<grid_of(n3), 256, 0, s>>>(c->g_val[1].p, n3, c->g_val[0].p);
        B2_KERNEL_CHECK();
    }
    const uint64_t *ekey = c->g_key[1].p;
    const uint32_t *eval = c->g_val[1].p, *einv = c->g_val[0].p;
    {
        // per face: 3 inverse entries, the three runs (about 2 keys + 2 values each on a manifold mesh), one count
        ScopedTimer t(c, "graph_adj_count", (12.0 + 3 * (2 * 8 + 2 * 4) + 4.0) * F + 4.0 * (F + 1) * 2);
        B2_LAUNCH k_graph_adj_count<<<grid, 256, 0, s>>>(ekey, eval, einv, F, c->g_cnt.p, c->g_scal.p);
        B2_KERNEL_CHECK();
        B2_TRY(cub_exclusive_sum_u32(c, c->g_cnt.p, c->adj_ptr.p, (size_t)F + 1));
    }
    unsigned long long sc[8];
    uint32_t num_adj = 0;
    B2_CUDA(cudaMemcpyAsync(sc, c->g_scal.p, sizeof(sc), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaMemcpyAsync(&num_adj, c->adj_ptr.p + F, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaStreamSynchronize(s));
    // sum of the rows = sum min(n, 3) + sum max(n - 3, 0) <= 3F + scal[3]: below 2^32 the u32 offsets cannot wrap
    if (3ull * F + sc[3] > 0xFFFFFFFFull) {
        set_error("build_mesh_graph: the face adjacency has more than 2^32 - 1 entries");
        return B2TEX_ERR_LIMITS;
    }
    B2_TRY(c->adj_idx.alloc(num_adj));
    {
        ScopedTimer t(c, "graph_adj_fill", (12.0 + 3 * (2 * 8 + 2 * 4) + 4.0) * F + 4.0 * num_adj);
        B2_LAUNCH k_graph_adj_fill<<<grid, 256, 0, s>>>(ekey, eval, einv, F, c->adj_ptr.p, c->adj_idx.p);
        B2_KERNEL_CHECK();
    }

    // ---- vertex -> faces ----
    B2_TRY(c->vf_idx.alloc(n3));
    {
        ScopedTimer t(c, "graph_vf", 4.0 * n3 + ((bits + 7) / 8) * 2.0 * 8 * n3 + 4.0 * n3 + 4.0 * (nv + 1));
        B2_LAUNCH k_graph_corner_faces<<<grid_of(n3), 256, 0, s>>>(n3, c->g_val[0].p);
        B2_KERNEL_CHECK();
        size_t tb = 0;
        B2_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, c->faces.p, c->g_val[1].p, c->g_val[0].p, c->vf_idx.p,
                                                (int)n3, 0, bits, s));
        B2_TRY(c->cub_tmp.alloc(tb));
        B2_CUDA(cub::DeviceRadixSort::SortPairs(c->cub_tmp.p, tb, c->faces.p, c->g_val[1].p, c->g_val[0].p, c->vf_idx.p,
                                                (int)n3, 0, bits, s));
        B2_LAUNCH k_graph_ring_ptr<<<grid_of(n3 + 1), 256, 0, s>>>(c->g_val[1].p, n3, nv, c->vf_ptr.p);
        B2_KERNEL_CHECK();
    }

    // ---- vertex -> vertices ----
    B2_TRY(c->vv_idx.alloc(n6));   // an upper bound; n is set to the distinct count below
    uint32_t *vv_pos = (uint32_t *)c->g_key[0].p;   // the unsorted keys are dead after the sort
    {
        ScopedTimer t(c, "graph_vv", 12.0 * n3 + 8.0 * n6 + passes * vv_pass_bytes + 8.0 * n6 + 4.0 * n6 +
                                         2 * 4.0 * n6 + 12.0 * n6 + 4.0 * (nv + 1));
        B2_LAUNCH k_graph_directed_keys<<<grid_of(n3), 256, 0, s>>>(c->faces.p, n3, bits, c->g_key[0].p);
        B2_KERNEL_CHECK();
        size_t tb = 0;
        B2_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, c->g_key[0].p, c->g_key[1].p, (int)n6, 0, ebits, s));
        B2_TRY(c->cub_tmp.alloc(tb));
        B2_CUDA(cub::DeviceRadixSort::SortKeys(c->cub_tmp.p, tb, c->g_key[0].p, c->g_key[1].p, (int)n6, 0, ebits, s));
        B2_LAUNCH k_graph_run_heads<<<grid_of(n6), 256, 0, s>>>(c->g_key[1].p, n6, c->g_cnt.p);
        B2_KERNEL_CHECK();
        B2_TRY(cub_exclusive_sum_u32(c, c->g_cnt.p, vv_pos, n6));
        B2_LAUNCH k_graph_vv_scatter<<<grid_of(n6 + 1), 256, 0, s>>>(c->g_key[1].p, c->g_cnt.p, vv_pos, n6, bits, nv,
                                                                     c->vv_ptr.p, c->vv_idx.p, c->g_scal.p);
        B2_KERNEL_CHECK();
    }
    B2_CUDA(cudaMemcpyAsync(sc, c->g_scal.p, sizeof(sc), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaStreamSynchronize(s));
    c->vv_idx.n = (size_t)sc[4];
    mark_valid(c, ADJ | RINGS);
    if (info) {
        info->num_adjacency = num_adj;
        info->num_vertex_faces = n3;
        info->num_vertex_neighbours = (uint32_t)sc[4];
        info->max_face_degree = (uint32_t)sc[1];
        info->num_non_manifold_edges = (uint32_t)sc[2];
    }
    return B2TEX_OK;
}

int validate_faces(b2tex_ctx *c, const uint32_t *faces, uint32_t F, uint32_t nv, const char *fn, const char *timer)
{
    cudaStream_t s = c->stream;
    const unsigned grid = (unsigned)std::min<size_t>(((size_t)F + 1 + 255) / 256 + 1, (size_t)c->num_sms * 16);
    B2_TRY(c->g_scal.alloc(8));
    unsigned long long init[8] = {GRAPH_NONE, 0, 0, 0, 0, 0, 0, 0};
    B2_CUDA(cudaMemcpyAsync(c->g_scal.p, init, sizeof(init), cudaMemcpyHostToDevice, s));
    {
        ScopedTimer t(c, timer, 12.0 * F);
        if (F) B2_LAUNCH k_graph_validate<<<grid, 256, 0, s>>>(faces, F, nv, c->g_scal.p);
        B2_KERNEL_CHECK();
    }
    unsigned long long bad = GRAPH_NONE;
    B2_CUDA(cudaMemcpyAsync(&bad, c->g_scal.p, sizeof(bad), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaStreamSynchronize(s));
    if (bad != GRAPH_NONE) {
        uint32_t fv[3];
        B2_CUDA(cudaMemcpyAsync(fv, faces + 3 * (size_t)bad, sizeof(fv), cudaMemcpyDeviceToHost, s));
        B2_CUDA(cudaStreamSynchronize(s));
        set_error("%s: face %llu (%u %u %u) has a vertex index >= %u vertices", fn, bad, fv[0], fv[1], fv[2], nv);
        return B2TEX_ERR_ARG;
    }
    return B2TEX_OK;
}

}  // namespace b2
