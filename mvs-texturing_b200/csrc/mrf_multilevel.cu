// mrf_multilevel.cu -- the contraction step of multilevel view selection (mapMAP's use_multilevel,
// view_selection.cpp:103-115), the schedule defined in oracle/mrf_multilevel.c and reproduced here bit for bit.
//
// A labeling is contracted into a coarse MRF: one node per connected component of the face graph restricted to edges
// whose two faces carry the same label (a "region").  mrf.cu then runs the forest BCD on it with weighted Potts terms and
// projects the coarse labels back through mrf_project.  The coarse MRF lives in grow-only context scratch (ml_*).
//
//   components : min-id hooking + pointer jumping, repeated until no same-label edge joins two trees.  Every parent pointer
//                points to a lower face, so the root of a component is its lowest face, whatever order the threads ran in.
//   numbering  : scan of the root flags -> node ids in the order of the lowest face; node size by integer atomics
//   label lists: (node << 16 | view) keys of every candidate of every face, stable radix sort with the candidate index as
//                value (so a run lists the members in ascending face order); a run whose length is the node size is in
//                every member's list (one load decides it).  Its cost is summed sequentially along the run from 0.0f
//                (oracle order), one thread per kept run.
//   edges      : (node << 32 | node') keys of every fine adjacency entry that crosses two nodes, sorted; each run is one
//                coarse CSR entry whose weight is the run length (an integer, exact in fp32).  Rows come out ascending.
// CUB only for the radix sorts and the scans, as in graph.cu.
#include <cub/cub.cuh>

#include "common.cuh"

namespace b2 {
namespace {

inline unsigned grid_for(size_t n) { return (unsigned)std::max<size_t>(1, (n + 255) / 256); }
inline int bits_for(uint64_t n) { int b = 0; while (b < 64 && (n >> b)) ++b; return std::max(b, 1); }
// elements of each u32 scratch buffer (ml_u32[0..2]): per face + 1 in the component phase (comp, root flags and their
// scan), per candidate + 1 for the label lists, per adjacency entry + 1 for the edges
inline size_t contract_u32_elems(uint32_t F, uint64_t nnz, uint32_t A) { return std::max(std::max((size_t)F, (size_t)nnz), (size_t)A) + 1; }

__global__ void __launch_bounds__(256) k_ml_comp_init(uint32_t F, uint32_t *comp)
{
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v < F) comp[v] = v;
}

// every same-label edge whose endpoints sit in different trees links the higher root below the lower one
__global__ void __launch_bounds__(256) k_ml_hook(uint32_t F, const uint32_t *__restrict__ adj_ptr, const uint32_t *__restrict__ adj_idx,
                                                 const uint32_t *__restrict__ labels, uint32_t *comp, uint32_t *changed)
{
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= F) return;
    const uint32_t lv = labels[v];
    bool ch = false;
    for (uint32_t a = adj_ptr[v]; a < adj_ptr[v + 1]; ++a) {
        const uint32_t w = adj_idx[a];
        if (w <= v || labels[w] != lv) continue;   // each undirected edge once
        const uint32_t pv = __ldcg(comp + v), pw = __ldcg(comp + w);
        if (pv == pw) continue;
        atomicMin(comp + max(pv, pw), min(pv, pw));
        ch = true;
    }
    if (ch) *changed = 1u;
}

__global__ void __launch_bounds__(256) k_ml_jump(uint32_t F, uint32_t *comp)
{
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= F) return;
    uint32_t p = __ldcg(comp + v);
    for (uint32_t q = __ldcg(comp + p); q != p; q = __ldcg(comp + p)) p = q;
    comp[v] = p;
}

__global__ void __launch_bounds__(256) k_ml_root_flags(uint32_t F, const uint32_t *__restrict__ comp, uint32_t *flag)
{
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v < F) flag[v] = comp[v] == v ? 1u : 0u;
    if (v == F) flag[v] = 0u;
}

// region[v] = node of v's root; the root also writes the node's label; node sizes by atomics
__global__ void __launch_bounds__(256) k_ml_region(uint32_t F, const uint32_t *__restrict__ comp, const uint32_t *__restrict__ rid,
                                                   const uint32_t *__restrict__ labels, uint32_t *region, uint32_t *clabels,
                                                   uint32_t *csize)
{
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= F) return;
    const uint32_t r = rid[comp[v]];
    region[v] = r;
    if (comp[v] == v) clabels[r] = labels[v];
    atomicAdd(csize + r, 1u);
}

__global__ void __launch_bounds__(256) k_ml_label_keys(uint32_t F, const uint64_t *__restrict__ ptr, const uint16_t *__restrict__ view,
                                                       const uint32_t *__restrict__ region, uint64_t *key, uint32_t *val)
{
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= F) return;
    const uint64_t r = (uint64_t)region[v] << 16;
    for (uint64_t k = ptr[v]; k < ptr[v + 1]; ++k) { key[k] = r | view[k]; val[k] = (uint32_t)k; }
}

// run heads of the sorted (node, view) keys: keep[i] = 1 where the run is as long as the node (the view is in every
// member's list), its cost summed along the run (ascending face order) into csum[i].  A run holds at most one entry per
// member, so one load at the node size's distance decides it without walking the run; only kept runs are summed, and their
// loads go out in batches of 16 ahead of the (sequential, oracle-order) additions.
__global__ void __launch_bounds__(256) k_ml_label_runs(uint32_t n, const uint64_t *__restrict__ key, const uint32_t *__restrict__ val,
                                                       const float *__restrict__ cost, const uint32_t *__restrict__ csize,
                                                       uint32_t *keep, float *csum)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == n) keep[i] = 0u;
    if (i >= n) return;
    const uint64_t k = key[i];
    uint32_t kp = 0u;
    if (i == 0 || key[i - 1] != k) {
        const uint32_t size = csize[k >> 16];
        if ((uint64_t)i + size <= n && key[i + size - 1] == k) {
            constexpr uint32_t B = 16;
            const uint32_t *vr = val + i;
            float s = 0.0f;
            uint32_t j = 0;
            for (; j + B <= size; j += B) {
                float c[B];
#pragma unroll
                for (uint32_t q = 0; q < B; ++q) c[q] = cost[vr[j + q]];
#pragma unroll
                for (uint32_t q = 0; q < B; ++q) s = s + c[q];
            }
            for (; j < size; ++j) s = s + cost[vr[j]];
            kp = 1u;
            csum[i] = s;
        }
    }
    keep[i] = kp;
}

__global__ void __launch_bounds__(256) k_ml_label_scatter(uint32_t n, const uint64_t *__restrict__ key, const uint32_t *__restrict__ keep,
                                                          const uint32_t *__restrict__ out, const float *__restrict__ csum,
                                                          uint16_t *cview, float *ccost, uint64_t *ccnt)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !keep[i]) return;
    const uint32_t o = out[i];
    cview[o] = (uint16_t)(key[i] & 0xFFFFu);
    ccost[o] = csum[i];
    atomicAdd(reinterpret_cast<unsigned long long *>(ccnt + (key[i] >> 16)), 1ull);
}

// position of every node's label in its list (0 for unseen nodes, whose list is empty)
__global__ void __launch_bounds__(256) k_ml_lidx(uint32_t n, const uint64_t *__restrict__ cptr, const uint16_t *__restrict__ cview,
                                                 const uint32_t *__restrict__ clabels, uint32_t *clidx)
{
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const uint64_t p0 = cptr[r];
    uint64_t lo = p0, hi = cptr[r + 1];
    const uint32_t lab = clabels[r];
    while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if ((uint32_t)cview[mid] + 1u < lab) lo = mid + 1; else hi = mid;
    }
    clidx[r] = lab ? (uint32_t)(lo - p0) : 0u;
}

// keys of the fine adjacency entries that cross two nodes; the others get `none`, which sorts last
__global__ void __launch_bounds__(256) k_ml_edge_keys(uint32_t F, const uint32_t *__restrict__ adj_ptr, const uint32_t *__restrict__ adj_idx,
                                                      const uint32_t *__restrict__ region, uint64_t none, uint64_t *key)
{
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= F) return;
    const uint64_t rv = region[v];
    for (uint32_t a = adj_ptr[v]; a < adj_ptr[v + 1]; ++a) {
        const uint32_t rw = region[adj_idx[a]];
        key[a] = rw != rv ? (rv << 32 | rw) : none;
    }
}

__global__ void __launch_bounds__(256) k_ml_edge_heads(uint32_t n, const uint64_t *__restrict__ key, uint64_t none, uint32_t *head)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == n) head[i] = 0u;
    if (i >= n) return;
    head[i] = key[i] != none && (i == 0 || key[i - 1] != key[i]) ? 1u : 0u;
}

__global__ void __launch_bounds__(256) k_ml_edge_scatter(uint32_t n, const uint64_t *__restrict__ key, const uint32_t *__restrict__ head,
                                                         const uint32_t *__restrict__ out, uint32_t *cidx, float *cw, uint32_t *cdeg)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !head[i]) return;
    const uint64_t k = key[i];
    uint32_t j = i + 1;
    while (j < n && key[j] == k) ++j;
    const uint32_t o = out[i];
    cidx[o] = (uint32_t)(k & 0xFFFFFFFFu);
    cw[o] = (float)(j - i);
    atomicAdd(cdeg + (k >> 32), 1u);
}

// labels[f] = coarse label of f's node, lidx[f] = its position in f's list; a no-op once the stop rule has fired
__global__ void __launch_bounds__(256) k_ml_project(uint32_t F, const uint32_t *__restrict__ region, const uint32_t *__restrict__ clabels,
                                                    const uint64_t *__restrict__ ptr, const uint16_t *__restrict__ view,
                                                    const uint32_t *stop, uint32_t *labels, uint32_t *lidx)
{
    if (__ldcg(stop)) return;
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= F) return;
    const uint32_t x = __ldcg(clabels + region[v]);
    const uint64_t p0 = ptr[v];
    uint64_t lo = p0, hi = ptr[v + 1];
    while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if ((uint32_t)view[mid] + 1u < x) lo = mid + 1; else hi = mid;
    }
    labels[v] = x;
    lidx[v] = x ? (uint32_t)(lo - p0) : 0u;
}

template <typename T>
int exclusive_sum(b2tex_ctx *c, const T *in, T *out, size_t n)
{
    size_t bytes = 0;
    B2_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, n, c->stream));
    B2_TRY(c->cub_tmp.alloc(bytes));
    B2_CUDA(cub::DeviceScan::ExclusiveSum(c->cub_tmp.p, bytes, in, out, n, c->stream));
    return B2TEX_OK;
}

}  // namespace

int mrf_contract(b2tex_ctx *c, uint32_t *num_nodes)
{
    cudaStream_t s = c->stream;
    const uint32_t F = c->F;
    const uint64_t nnz = c->nnz;
    uint32_t A = 0;
    B2_CUDA(cudaMemcpyAsync(&A, c->adj_ptr.p + F, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaStreamSynchronize(s));
    if (nnz >= 0x7FFFFFFFull || A >= 0x7FFFFFFFu || F >= 0x7FFFFFFFu) {
        set_error("multilevel view selection: more than 2^31 - 2 faces, candidates or adjacency entries");
        return B2TEX_ERR_LIMITS;
    }
    const size_t nk = std::max<size_t>(nnz, A), nu = contract_u32_elems(F, nnz, A);
    B2_TRY(c->ml_region.alloc(F));
    B2_TRY(c->ml_u32[0].alloc(nu)); B2_TRY(c->ml_u32[1].alloc(nu)); B2_TRY(c->ml_u32[2].alloc(nu));
    B2_TRY(c->ml_key[0].alloc(nk)); B2_TRY(c->ml_key[1].alloc(nk));
    B2_TRY(c->ml_f32.alloc(nk));
    B2_TRY(c->ml_changed.alloc(1));
    uint32_t *comp = c->ml_u32[0].p, *flag = c->ml_u32[1].p, *rid = c->ml_u32[2].p;

    // ---- components: hook + jump until stable (a handful of rounds: jumping halves every path) ----
    {
        ScopedTimer t(c, "mrf_ml.components");
        B2_LAUNCH k_ml_comp_init<<<grid_for(F), 256, 0, s>>>(F, comp);
        B2_KERNEL_CHECK();
        for (;;) {
            uint32_t changed = 0;
            B2_CUDA(cudaMemsetAsync(c->ml_changed.p, 0, sizeof(uint32_t), s));
            B2_LAUNCH k_ml_hook<<<grid_for(F), 256, 0, s>>>(F, c->adj_ptr.p, c->adj_idx.p, c->labels.p, comp, c->ml_changed.p);
            B2_LAUNCH k_ml_jump<<<grid_for(F), 256, 0, s>>>(F, comp);
            B2_KERNEL_CHECK();
            B2_CUDA(cudaMemcpyAsync(&changed, c->ml_changed.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
            B2_CUDA(cudaStreamSynchronize(s));
            if (!changed) break;
        }
    }
    // ---- node ids in the order of the lowest face ----
    uint32_t n = 0;
    {
        ScopedTimer t(c, "mrf_ml.numbering");
        B2_LAUNCH k_ml_root_flags<<<grid_for((size_t)F + 1), 256, 0, s>>>(F, comp, flag);
        B2_KERNEL_CHECK();
        B2_TRY(exclusive_sum<uint32_t>(c, flag, rid, (size_t)F + 1));
        B2_CUDA(cudaMemcpyAsync(&n, rid + F, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        B2_CUDA(cudaStreamSynchronize(s));
        B2_TRY(c->ml_clabels.alloc(n)); B2_TRY(c->ml_clidx.alloc(n)); B2_TRY(c->ml_csize.alloc(n));
        B2_TRY(c->ml_cptr.alloc((size_t)n + 1)); B2_TRY(c->ml_cadj_ptr.alloc((size_t)n + 1)); B2_TRY(c->ml_cadj4.alloc(n));
        B2_TRY(c->ml_csize.zero(s));
        B2_LAUNCH k_ml_region<<<grid_for(F), 256, 0, s>>>(F, comp, rid, c->labels.p, c->ml_region.p, c->ml_clabels.p, c->ml_csize.p);
        B2_KERNEL_CHECK();
    }
    const int nbits = bits_for(n);
    // ---- label lists: the intersection of the members' lists, costs summed in ascending face order ----
    {
        ScopedTimer t(c, "mrf_ml.label_lists");
        B2_TRY(c->ml_cview.alloc(nnz)); B2_TRY(c->ml_ccost.alloc(nnz));
        if (nnz) {
            B2_LAUNCH k_ml_label_keys<<<grid_for(F), 256, 0, s>>>(F, c->dc_ptr.p, c->dc_view.p, c->ml_region.p, c->ml_key[0].p, flag);
            B2_KERNEL_CHECK();
            size_t tb = 0;
            B2_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, c->ml_key[0].p, c->ml_key[1].p, flag, rid, (int)nnz, 0, 16 + nbits, s));
            B2_TRY(c->cub_tmp.alloc(tb));
            B2_CUDA(cub::DeviceRadixSort::SortPairs(c->cub_tmp.p, tb, c->ml_key[0].p, c->ml_key[1].p, flag, rid, (int)nnz, 0, 16 + nbits, s));
        }
        // the sorted candidate indices are in rid; comp and flag are free: keep flags in comp, output positions in flag
        B2_LAUNCH k_ml_label_runs<<<grid_for(nnz + 1), 256, 0, s>>>((uint32_t)nnz, c->ml_key[1].p, rid, c->dc_cost.p, c->ml_csize.p,
                                                                     comp, c->ml_f32.p);
        B2_KERNEL_CHECK();
        B2_TRY(exclusive_sum<uint32_t>(c, comp, flag, nnz + 1));
        uint64_t *ccnt = c->ml_cptr.p;
        B2_TRY(c->ml_cnt64.alloc((size_t)n + 1));
        B2_TRY(c->ml_cnt64.zero(s));
        B2_LAUNCH k_ml_label_scatter<<<grid_for(nnz), 256, 0, s>>>((uint32_t)nnz, c->ml_key[1].p, comp, flag, c->ml_f32.p,
                                                                    c->ml_cview.p, c->ml_ccost.p, c->ml_cnt64.p);
        B2_KERNEL_CHECK();
        B2_TRY(exclusive_sum<uint64_t>(c, c->ml_cnt64.p, ccnt, (size_t)n + 1));
        B2_LAUNCH k_ml_lidx<<<grid_for(n), 256, 0, s>>>(n, ccnt, c->ml_cview.p, c->ml_clabels.p, c->ml_clidx.p);
        B2_KERNEL_CHECK();
    }
    // ---- edges: one coarse entry per (node, node') run, weight = the run length ----
    {
        ScopedTimer t(c, "mrf_ml.edges");
        const uint64_t none = (uint64_t)n << 32;   // above every real key, inside 32 + nbits bits
        B2_TRY(c->ml_cadj_idx.alloc(A)); B2_TRY(c->ml_cwgt.alloc(A));
        B2_TRY(c->ml_cdeg.alloc((size_t)n + 1));
        B2_TRY(c->ml_cdeg.zero(s));
        if (A) {
            B2_LAUNCH k_ml_edge_keys<<<grid_for(F), 256, 0, s>>>(F, c->adj_ptr.p, c->adj_idx.p, c->ml_region.p, none, c->ml_key[0].p);
            B2_KERNEL_CHECK();
            size_t tb = 0;
            B2_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, c->ml_key[0].p, c->ml_key[1].p, (int)A, 0, 32 + nbits, s));
            B2_TRY(c->cub_tmp.alloc(tb));
            B2_CUDA(cub::DeviceRadixSort::SortKeys(c->cub_tmp.p, tb, c->ml_key[0].p, c->ml_key[1].p, (int)A, 0, 32 + nbits, s));
        }
        B2_LAUNCH k_ml_edge_heads<<<grid_for((size_t)A + 1), 256, 0, s>>>(A, c->ml_key[1].p, none, comp);
        B2_KERNEL_CHECK();
        B2_TRY(exclusive_sum<uint32_t>(c, comp, flag, (size_t)A + 1));
        B2_LAUNCH k_ml_edge_scatter<<<grid_for(A), 256, 0, s>>>(A, c->ml_key[1].p, comp, flag, c->ml_cadj_idx.p, c->ml_cwgt.p,
                                                                c->ml_cdeg.p);
        B2_KERNEL_CHECK();
        B2_TRY(exclusive_sum<uint32_t>(c, c->ml_cdeg.p, c->ml_cadj_ptr.p, (size_t)n + 1));
    }
    c->ml_nodes = n;
    *num_nodes = n;
    return B2TEX_OK;
}

int mrf_project(b2tex_ctx *c, const uint32_t *stop)
{
    const uint32_t F = c->F;
    B2_LAUNCH k_ml_project<<<grid_for(F), 256, 0, c->stream>>>(F, c->ml_region.p, c->ml_clabels.p, c->dc_ptr.p, c->dc_view.p, stop,
                                                               c->labels.p, c->mrf_lidx.p);
    B2_KERNEL_CHECK();
    return B2TEX_OK;
}

}  // namespace b2
