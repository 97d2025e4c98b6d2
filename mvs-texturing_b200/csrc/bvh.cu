// bvh.cu -- K2: LBVH build on the device (Morton sort + Karras hierarchy + bottom-up refit).
// Stands where the reference builds rayint's acc::BVHTree (calculate_data_costs.cpp:144).
// CUB is used for the key sort only (plumbing); everything else is hand written.
#include <cub/cub.cuh>

#include "common.cuh"

namespace b2 {

namespace {

__device__ __forceinline__ uint32_t f2ord(float f)
{
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float ord2f(uint32_t o)
{
    uint32_t u = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f; memcpy(&f, &u, 4); return f;
#endif
}

__global__ void k_bounds_init(uint32_t *b)
{
    if (threadIdx.x < 3) b[threadIdx.x] = 0xFFFFFFFFu;
    else if (threadIdx.x < 6) b[threadIdx.x] = 0u;
}

__global__ void k_bounds(const float *__restrict__ verts, uint32_t nv, uint32_t *b)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t lo[3] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu}, hi[3] = {0, 0, 0};
    for (; i < nv; i += gridDim.x * blockDim.x)
        for (int k = 0; k < 3; ++k) {
            uint32_t o = f2ord(verts[3 * (size_t)i + k]);
            lo[k] = min(lo[k], o);
            hi[k] = max(hi[k], o);
        }
    for (int k = 0; k < 3; ++k) {
        for (int s = 16; s; s >>= 1) {
            lo[k] = min(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], s));
            hi[k] = max(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], s));
        }
        if ((threadIdx.x & 31) == 0) { atomicMin(&b[k], lo[k]); atomicMax(&b[3 + k], hi[k]); }
    }
}

__device__ __forceinline__ uint64_t expand21(uint64_t v)
{
    v &= 0x1FFFFFull;
    v = (v | v << 32) & 0x1F00000000FFFFull;
    v = (v | v << 16) & 0x1F0000FF0000FFull;
    v = (v | v << 8) & 0x100F00F00F00F00Full;
    v = (v | v << 4) & 0x10C30C30C30C30C3ull;
    v = (v | v << 2) & 0x1249249249249249ull;
    return v;
}

__global__ void k_morton(const float *__restrict__ verts, const uint32_t *__restrict__ faces, uint32_t nf,
                         const uint32_t *__restrict__ bnd, uint64_t *keys, uint32_t *ids)
{
    uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nf) return;
    float lo[3], ext[3];
    for (int k = 0; k < 3; ++k) {
        lo[k] = ord2f(bnd[k]);
        ext[k] = ord2f(bnd[3 + k]) - lo[k];
        if (!(ext[k] > 0.0f)) ext[k] = 1.0f;
    }
    uint64_t code = 0;
    for (int k = 0; k < 3; ++k) {
        float a = verts[3 * (size_t)faces[3 * (size_t)f] + k];
        float b = verts[3 * (size_t)faces[3 * (size_t)f + 1] + k];
        float c = verts[3 * (size_t)faces[3 * (size_t)f + 2] + k];
        float cen = (fminf(a, fminf(b, c)) + fmaxf(a, fmaxf(b, c))) * 0.5f;
        float t = (cen - lo[k]) / ext[k];
        t = fminf(fmaxf(t, 0.0f), 1.0f);
        uint64_t q = (uint64_t)(t * 2097151.0f);
        code |= expand21(q) << (2 - k);
    }
    keys[f] = code;
    ids[f] = f;
}

// Morton keys of the vertices (for coherent visibility rays)
__global__ void k_morton_verts(const float *__restrict__ verts, uint32_t nv, const uint32_t *__restrict__ bnd,
                               uint64_t *keys, uint32_t *ids)
{
    uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nv) return;
    uint64_t code = 0;
    for (int k = 0; k < 3; ++k) {
        float lo = ord2f(bnd[k]), ext = ord2f(bnd[3 + k]) - lo;
        if (!(ext > 0.0f)) ext = 1.0f;
        float t = fminf(fmaxf((verts[3 * (size_t)v + k] - lo) / ext, 0.0f), 1.0f);
        code |= expand21((uint64_t)(t * 2097151.0f)) << (2 - k);
    }
    keys[v] = code;
    ids[v] = v;
}

__global__ void k_invert_perm(const uint32_t *__restrict__ order, uint32_t n, uint32_t *rank)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) rank[order[i]] = i;
}

__global__ void k_gather_tris(const float *__restrict__ verts, const uint32_t *__restrict__ faces,
                              const uint32_t *__restrict__ ids, uint32_t nf, float *tri)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nf) return;
    uint32_t f = ids[i];
    for (int c = 0; c < 3; ++c) {
        const float *v = verts + 3 * (size_t)faces[3 * (size_t)f + c];
        tri[9 * (size_t)i + 3 * c + 0] = v[0];
        tri[9 * (size_t)i + 3 * c + 1] = v[1];
        tri[9 * (size_t)i + 3 * c + 2] = v[2];
    }
}

__device__ __forceinline__ int delta(const uint64_t *__restrict__ keys, int n, int i, int j)
{
    if (j < 0 || j >= n) return -1;
    uint64_t a = keys[i], b = keys[j];
    if (a == b) return 64 + __clz((uint32_t)i ^ (uint32_t)j);
    return __clzll((long long)(a ^ b));
}

// Karras 2012: one thread per internal node
__global__ void k_hierarchy(const uint64_t *__restrict__ keys, int n, BvhNode *nodes, int *parent_internal,
                            int *parent_leaf)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n - 1) return;
    int d = (delta(keys, n, i, i + 1) - delta(keys, n, i, i - 1)) >= 0 ? 1 : -1;
    int dmin = delta(keys, n, i, i - d);
    int lmax = 2;
    while (delta(keys, n, i, i + lmax * d) > dmin) lmax *= 2;
    int l = 0;
    for (int t = lmax / 2; t >= 1; t /= 2)
        if (delta(keys, n, i, i + (l + t) * d) > dmin) l += t;
    int j = i + l * d;
    int dnode = delta(keys, n, i, j);
    int s = 0;
    int t = l;
    do {
        t = (t + 1) >> 1;
        if (delta(keys, n, i, i + (s + t) * d) > dnode) s += t;
    } while (t > 1);
    int gamma = i + s * d + min(d, 0);
    int lo = min(i, j), hi = max(i, j);
    int left = (lo == gamma) ? ~gamma : gamma;
    int right = (hi == gamma + 1) ? ~(gamma + 1) : gamma + 1;
    nodes[i].left = left;
    nodes[i].right = right;
    nodes[i].pad0 = nodes[i].pad1 = 0;
    if (left < 0) parent_leaf[~left] = i; else parent_internal[left] = i;
    if (right < 0) parent_leaf[~right] = i; else parent_internal[right] = i;
    if (i == 0) parent_internal[0] = -1;
}

__device__ __forceinline__ void tri_box(const float *t9, float pad, float *lo, float *hi)
{
    for (int k = 0; k < 3; ++k) {
        lo[k] = fminf(t9[k], fminf(t9[3 + k], t9[6 + k])) - pad;
        hi[k] = fmaxf(t9[k], fmaxf(t9[3 + k], t9[6 + k])) + pad;
    }
}

// bottom-up refit: the second thread to arrive at a node computes it
__global__ void k_refit(BvhNode *nodes, const int *__restrict__ parent_internal,
                        const int *__restrict__ parent_leaf, const float *__restrict__ tri, int n,
                        float pad, uint32_t *counters, float *node_box /* 6 per internal node */)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float lo[3], hi[3];
    tri_box(tri + 9 * (size_t)i, pad, lo, hi);
    int node = parent_leaf[i];
    int child = ~i;
    while (node >= 0) {
        BvhNode *nd = &nodes[node];
        if (nd->left == child) {
            for (int k = 0; k < 3; ++k) { nd->lo0[k] = lo[k]; nd->hi0[k] = hi[k]; }
        } else {
            for (int k = 0; k < 3; ++k) { nd->lo1[k] = lo[k]; nd->hi1[k] = hi[k]; }
        }
        __threadfence();
        if (atomicAdd(&counters[node], 1u) == 0u) return;  // first arrival: sibling not ready
        __threadfence();
        volatile BvhNode *vn = nd;
        for (int k = 0; k < 3; ++k) {
            lo[k] = fminf(vn->lo0[k], vn->lo1[k]);
            hi[k] = fmaxf(vn->hi0[k], vn->hi1[k]);
        }
        child = node;
        node = parent_internal[node];
    }
    (void)node_box;
}

}  // namespace

int build_bvh(b2tex_ctx *c, bool force)
{
    if ((c->valid & BVH) && !force) return B2TEX_OK;
    invalidate(c, BVH);
    ScopedTimer tm(c, "bvh_build");
    cudaStream_t s = c->stream;
    const uint32_t n = c->F;
    c->bvh.num_tris = n;
    if (n == 0) { mark_valid(c, BVH); return B2TEX_OK; }

    DevBuf<uint32_t> &bnd = c->s_bnd, &ids_in = c->s_ids_in, &ids_out = c->s_ids_out, &counters = c->s_counters;
    DevBuf<uint64_t> &keys_in = c->s_keys_in, &keys_out = c->s_keys_out;
    DevBuf<int> &parent_internal = c->s_parent_internal, &parent_leaf = c->s_parent_leaf;
    B2_TRY(bnd.alloc(8));
    B2_LAUNCH k_bounds_init<<<1, 32, 0, s>>>(bnd.p);
    B2_LAUNCH k_bounds<<<std::max(1, c->num_sms * 4), 256, 0, s>>>(c->verts.p, c->Vn, bnd.p);
    B2_KERNEL_CHECK();
    uint32_t hb[6];
    B2_CUDA(cudaMemcpyAsync(hb, bnd.p, sizeof(hb), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaStreamSynchronize(s));
    float ext[3];
    for (int k = 0; k < 3; ++k) ext[k] = ord2f(hb[3 + k]) - ord2f(hb[k]);
    float diag = sqrtf(ext[0] * ext[0] + ext[1] * ext[1] + ext[2] * ext[2]);
    float pad = 1e-5f * diag;  // same conservative padding as oracle/bvh.c

    // vertex order for the ray bitmaps
    {
        const uint32_t nv = c->Vn;
        DevBuf<uint64_t> &vk_in = c->s_vk_in, &vk_out = c->s_vk_out;
        DevBuf<uint32_t> &vi_in = c->s_vi_in;
        B2_TRY(vk_in.alloc(nv)); B2_TRY(vk_out.alloc(nv)); B2_TRY(vi_in.alloc(nv));
        B2_TRY(c->vorder.alloc(nv)); B2_TRY(c->vrank.alloc(nv));
        B2_LAUNCH k_morton_verts<<<(nv + 255) / 256, 256, 0, s>>>(c->verts.p, nv, bnd.p, vk_in.p, vi_in.p);
        size_t vb = 0;
        B2_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, vb, vk_in.p, vk_out.p, vi_in.p, c->vorder.p, (int)nv, 0, 63, s));
        B2_TRY(c->cub_tmp.alloc(vb));
        B2_CUDA(cub::DeviceRadixSort::SortPairs(c->cub_tmp.p, vb, vk_in.p, vk_out.p, vi_in.p, c->vorder.p, (int)nv, 0, 63, s));
        B2_LAUNCH k_invert_perm<<<(nv + 255) / 256, 256, 0, s>>>(c->vorder.p, nv, c->vrank.p);
        B2_KERNEL_CHECK();
    }
    B2_TRY(keys_in.alloc(n)); B2_TRY(keys_out.alloc(n));
    B2_TRY(ids_in.alloc(n)); B2_TRY(ids_out.alloc(n));
    B2_LAUNCH k_morton<<<(n + 255) / 256, 256, 0, s>>>(c->verts.p, c->faces.p, n, bnd.p, keys_in.p, ids_in.p);
    B2_KERNEL_CHECK();
    size_t tmp_bytes = 0;
    B2_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys_in.p, keys_out.p, ids_in.p, ids_out.p,
                                            (int)n, 0, 63, s));
    B2_TRY(c->cub_tmp.alloc(tmp_bytes));
    B2_CUDA(cub::DeviceRadixSort::SortPairs(c->cub_tmp.p, tmp_bytes, keys_in.p, keys_out.p, ids_in.p,
                                            ids_out.p, (int)n, 0, 63, s));
    B2_TRY(c->bvh.tri.alloc(9 * (size_t)n));
    B2_LAUNCH k_gather_tris<<<(n + 255) / 256, 256, 0, s>>>(c->verts.p, c->faces.p, ids_out.p, n, c->bvh.tri.p);
    B2_KERNEL_CHECK();
    if (n >= 2) {
        B2_TRY(c->bvh.nodes.alloc(n - 1));
        B2_TRY(parent_internal.alloc(n)); B2_TRY(parent_leaf.alloc(n));
        B2_TRY(counters.alloc(n)); B2_TRY(counters.zero(s));
        B2_LAUNCH k_hierarchy<<<(n - 1 + 255) / 256, 256, 0, s>>>(keys_out.p, (int)n, c->bvh.nodes.p, parent_internal.p,
                                                        parent_leaf.p);
        B2_LAUNCH k_refit<<<(n + 255) / 256, 256, 0, s>>>(c->bvh.nodes.p, parent_internal.p, parent_leaf.p, c->bvh.tri.p,
                                                (int)n, pad, counters.p, nullptr);
        B2_KERNEL_CHECK();
    }
    B2_CUDA(cudaStreamSynchronize(s));
    mark_valid(c, BVH);
    return B2TEX_OK;
}

}  // namespace b2
