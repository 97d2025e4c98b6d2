// seam.cu -- K8/K9: global seam leveling on the device.
//
// Replaces tex::global_seam_leveling up to the per-(vertex,label) adjust values
// (libs/tex/global_seam_leveling.cpp:140-291):
//   K8 assembly : unknown numbering (:156-176), Lhs = A^T A + Gamma^T Gamma built directly as a
//                 weighted graph Laplacian in CSR (no triplets, no sparse product; :182-249),
//                 b from seam-edge colour sampling (:26-43, :86-138), Rhs = A^T b (:266-270)
//   K9 solve    : Jacobi-preconditioned CG for the 3 colour channels at once, restating Eigen's
//                 conjugate_gradient() (:257-277) as ONE persistent cooperative kernel: CSR SpMV with
//                 the three right-hand sides packed in a float4, fused vector updates, grid-wide
//                 deterministic reductions, per-channel convergence, mean subtraction (:277).
// Colour source: whole view image of the label (see oracle/seam.c header; stage-isolated mode).
#include <cooperative_groups.h>
#include <math.h>

#include <memory>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace b2 {

namespace {

constexpr int MAXL = 64;  // labels per vertex kept (same cap as the oracle)

template <bool FILL>
__global__ void k_vertex_labels(uint32_t Vn, const uint32_t *__restrict__ vf_ptr,
                                const uint32_t *__restrict__ vf_idx, const uint32_t *__restrict__ labels,
                                uint32_t *cnt, const uint32_t *__restrict__ row_ptr, uint32_t *row_label,
                                uint32_t *row_vertex, uint32_t *limit_flags)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Vn) return;
    uint32_t tmp[MAXL];
    uint32_t n = 0;
    for (uint32_t a = vf_ptr[i]; a < vf_ptr[i + 1]; ++a) {
        uint32_t l = labels[vf_idx[a]];
        if (l == 0) continue;
        uint32_t k = 0;
        while (k < n && tmp[k] != l) ++k;
        if (k < n) continue;
        if (n >= MAXL) { atomicOr(limit_flags, 1u); continue; }   // the reference has no such cap: reported, not dropped silently
        uint32_t p = n++;
        while (p > 0 && tmp[p - 1] > l) { tmp[p] = tmp[p - 1]; --p; }
        tmp[p] = l;
    }
    if (!FILL) { cnt[i] = n; return; }
    uint32_t o = row_ptr[i];
    for (uint32_t k = 0; k < n; ++k) { row_label[o + k] = tmp[k]; row_vertex[o + k] = i; }
}

struct SeamMesh {
    const float *verts;
    const uint32_t *faces, *vf_ptr, *vf_idx, *vv_ptr, *vv_idx, *labels, *row_ptr, *row_label;
    const ViewDev *views;
};

__device__ __forceinline__ bool face_has_vertex(const uint32_t *__restrict__ faces, uint32_t f, uint32_t v)
{
    return faces[3 * (size_t)f] == v || faces[3 * (size_t)f + 1] == v || faces[3 * (size_t)f + 2] == v;
}

__device__ __forceinline__ void pixel_coords(const ViewDev &V, const float *X, float out[2])
{
    float cam[3], pix[3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
        cam[i] = (((0.0f + V.w2c[4 * i] * X[0]) + V.w2c[4 * i + 1] * X[1]) + V.w2c[4 * i + 2] * X[2])
            + 1.0f * V.w2c[4 * i + 3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
        pix[i] = ((0.0f + V.proj[3 * i] * cam[0]) + V.proj[3 * i + 1] * cam[1]) + V.proj[3 * i + 2] * cam[2];
    out[0] = pix[0] / pix[2] - 0.5f;
    out[1] = pix[1] / pix[2] - 0.5f;
}

// FloatImage::linear_at on bytes/255 (texture_patch.cpp:162-169)
__device__ __forceinline__ void sample_view(const ViewDev &V, float x, float y, float out[3])
{
    const int w = V.w, h = V.h;
    x = fmaxf(0.0f, fminf((float)(w - 1), x));
    y = fmaxf(0.0f, fminf((float)(h - 1), y));
    int fx = (int)x, fy = (int)y;
    int fx1 = min(fx + 1, w - 1), fy1 = min(fy + 1, h - 1);
    float w1 = x - (float)fx, w0 = 1.0f - w1;
    float w3 = y - (float)fy, w2 = 1.0f - w3;
    const uint8_t *a = V.rgb + 3 * ((size_t)fx + (size_t)fy * w);
    const uint8_t *b = V.rgb + 3 * ((size_t)fx1 + (size_t)fy * w);
    const uint8_t *c = V.rgb + 3 * ((size_t)fx + (size_t)fy1 * w);
    const uint8_t *d = V.rgb + 3 * ((size_t)fx1 + (size_t)fy1 * w);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch)
        out[ch] = (((float)a[ch] / 255.0f) * (w0 * w2) + ((float)b[ch] / 255.0f) * (w1 * w2))
            + ((float)c[ch] / 255.0f) * (w0 * w3) + ((float)d[ch] / 255.0f) * (w1 * w3);
}

// global_seam_leveling.cpp:26-43
__device__ void sample_edge(const ViewDev &V, const float p1[2], const float p2[2], float out[3])
{
    float p12[2] = {p2[0] - p1[0], p2[1] - p1[1]};
    float nrm = sqrtf((0.0f + p12[0] * p12[0]) + p12[1] * p12[1]);
    unsigned long long num_samples = (unsigned long long)(fmaxf(nrm, 1.0f) * 2.0f);
    float acc[3] = {0.0f, 0.0f, 0.0f}, wsum = 0.0f;
    for (unsigned long long s = 0; s < num_samples; ++s) {
        float fraction = (float)s / (float)(num_samples - 1);
        float col[3];
        sample_view(V, p1[0] + p12[0] * fraction, p1[1] + p12[1] * fraction, col);
        float wgt = 1.0f - fraction;
        for (int c = 0; c < 3; ++c) acc[c] += col[c] * wgt;
        wsum += wgt;
    }
    for (int c = 0; c < 3; ++c) out[c] = acc[c] / wsum;
}

// A rows of one vertex: label pairs l1<l2 with >= 1 seam edge (:214-237); FILL also computes b.
template <bool FILL>
__global__ void k_arows(uint32_t Vn, SeamMesh m, uint32_t *cnt, const uint32_t *__restrict__ arow_ptr,
                        uint32_t *arow_rows, float *arow_b, uint32_t *limit_flags)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Vn) return;
    uint32_t r0 = m.row_ptr[i], r1 = m.row_ptr[i + 1];
    uint32_t n = 0;
    if (r1 - r0 >= 2) {
        const float *v1 = m.verts + 3 * (size_t)i;
        for (uint32_t j = r0; j < r1; ++j)
            for (uint32_t k = j + 1; k < r1; ++k) {  // labels ascending => label1 < label2
                uint32_t label1 = m.row_label[j], label2 = m.row_label[k];
                float c1[3] = {0, 0, 0}, c2[3] = {0, 0, 0}, w1 = 0.0f, w2 = 0.0f;
                bool any = false;
                for (uint32_t a = m.vv_ptr[i]; a < m.vv_ptr[i + 1]; ++a) {
                    uint32_t adj = m.vv_idx[a];
                    if (adj == i) continue;
                    uint32_t ef[16], nef = 0;
                    for (uint32_t q = m.vf_ptr[i]; q < m.vf_ptr[i + 1]; ++q)
                        if (face_has_vertex(m.faces, m.vf_idx[q], adj)) {
                            if (nef < 16) ef[nef++] = m.vf_idx[q];
                            else atomicOr(limit_flags, 2u);   // more than 16 faces on one edge
                        }
                    for (uint32_t x = 0; x < nef; ++x)
                        for (uint32_t y = x + 1; y < nef; ++y) {
                            uint32_t fl1 = m.labels[ef[x]], fl2 = m.labels[ef[y]];
                            if (!(fl1 < fl2)) { uint32_t t = fl1; fl1 = fl2; fl2 = t; }
                            if (fl1 != label1 || fl2 != label2) continue;
                            const float *v2 = m.verts + 3 * (size_t)adj;
                            float d0 = v2[0] - v1[0], d1 = v2[1] - v1[1], d2 = v2[2] - v1[2];
                            float length = sqrtf(((0.0f + d0 * d0) + d1 * d1) + d2 * d2);
                            if (length == 0.0f) continue;
                            any = true;
                            if (FILL) {
                                float pa[2], pb[2], col[3];
                                const ViewDev &va = m.views[label1 - 1];
                                pixel_coords(va, v1, pa); pixel_coords(va, v2, pb);
                                sample_edge(va, pa, pb, col);
                                for (int c = 0; c < 3; ++c) c1[c] += col[c] * length;
                                w1 += length;
                                const ViewDev &vb = m.views[label2 - 1];
                                pixel_coords(vb, v1, pa); pixel_coords(vb, v2, pb);
                                sample_edge(vb, pa, pb, col);
                                for (int c = 0; c < 3; ++c) c2[c] += col[c] * length;
                                w2 += length;
                            }
                        }
                }
                if (!any) continue;
                if (FILL) {
                    uint32_t o = arow_ptr[i] + n;
                    arow_rows[2 * (size_t)o] = j;
                    arow_rows[2 * (size_t)o + 1] = k;
                    for (int c = 0; c < 3; ++c) arow_b[3 * (size_t)o + c] = c2[c] / w2 - c1[c] / w1;  // :131
                }
                ++n;
            }
    }
    if (!FILL) cnt[i] = n;
}

__device__ __forceinline__ uint32_t find_row(const SeamMesh &m, uint32_t v, uint32_t label)
{
    for (uint32_t k = m.row_ptr[v]; k < m.row_ptr[v + 1]; ++k)
        if (m.row_label[k] == label) return k;
    return 0xFFFFFFFFu;
}

// one thread per unknown: row of the weighted Laplacian, diag first
template <bool FILL>
__global__ void k_matrix(uint32_t R, SeamMesh m, const uint32_t *__restrict__ row_vertex,
                         const uint32_t *__restrict__ arow_ptr, const uint32_t *__restrict__ arow_rows,
                         const float *__restrict__ arow_b, uint32_t *cnt, const uint32_t *__restrict__ csr_ptr,
                         uint32_t *csr_col, float *csr_val, float *inv_diag, float *rhs /* [3][R] */,
                         uint32_t *csr_enc, float *diag_val)
{
    uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    const float lambda = 0.1f, lam2 = lambda * lambda;
    uint32_t i = row_vertex[r], label = m.row_label[r];
    uint32_t o = FILL ? csr_ptr[r] + 1 : 0;
    uint32_t n = 1;
    float gsum = 0.0f;
    uint32_t na = 0;
    for (uint32_t a = m.vv_ptr[i]; a < m.vv_ptr[i + 1]; ++a) {  // Gamma^T Gamma (:182-208)
        uint32_t adj = m.vv_idx[a];
        if (adj == i) continue;
        uint32_t c = find_row(m, adj, label);
        if (c == 0xFFFFFFFFu) continue;
        if (FILL) { csr_col[o] = c; csr_val[o] = -lam2; csr_enc[o] = c; ++o; }
        gsum += lam2;
        ++n;
    }
    float rh[3] = {0.0f, 0.0f, 0.0f};
    for (uint32_t a = arow_ptr[i]; a < arow_ptr[i + 1]; ++a) {  // A^T A (:211-237) and Rhs = A^T b
        uint32_t ra = arow_rows[2 * (size_t)a], rb = arow_rows[2 * (size_t)a + 1];
        if (ra != r && rb != r) continue;
        if (FILL) {
            csr_col[o] = (ra == r) ? rb : ra; csr_val[o] = -1.0f; csr_enc[o] = csr_col[o] | 0x80000000u; ++o;
            for (int c = 0; c < 3; ++c) {
                float b = arow_b[3 * (size_t)a + c];
                rh[c] = (ra == r) ? rh[c] + b : rh[c] - b;
            }
        }
        ++na;
        ++n;
    }
    if (!FILL) { cnt[r] = n; return; }
    float diag = (float)na + gsum;
    csr_col[csr_ptr[r]] = r;
    csr_val[csr_ptr[r]] = diag;
    csr_enc[csr_ptr[r]] = r;  // first entry of every row = the diagonal (value in diag_val)
    diag_val[r] = diag;
    inv_diag[r] = diag != 0.0f ? 1.0f / diag : 1.0f;  // Eigen DiagonalPreconditioner
    for (int c = 0; c < 3; ++c) rhs[(size_t)c * R + r] = rh[c];
}

// ---------------------------------------------------------------------------------------------
// K9: persistent cooperative Jacobi-PCG, 3 right-hand sides
// ---------------------------------------------------------------------------------------------
struct Pcg {
    uint32_t R;
    const uint32_t *csr_ptr, *csr_enc;  // enc = column | (weight class << 31): the Laplacian has only two
    const float *diag_val, *inv_diag, *rhs;  // off-diagonal values (-1 seam rows, -lambda^2 regulariser): 4 B per entry
    float *x, *r, *t;       // [3][R]
    float4 *p;              // [R] (x,y,z = channels)
    double *partials;       // [2][grid][8]
    uint32_t *status;       // [0..2] iterations, [3..5] residual bits, [6] loop iterations,
                            // [8..13] ns block 0 spent in SpMV / barrier A / update / barrier B / p update / loop-end barrier
    uint32_t max_iters;
    float tol;
    uint32_t timing;        // diagnostic (B2TEX_SEAM_TIMING): fill status[8..13]
};

__device__ __forceinline__ unsigned long long pcg_timer_ns()
{
#ifdef __CUDA_ARCH__
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
#else
    return 0ull;
#endif
}

// Sum of six doubles over the block in a fixed order: xor butterfly inside every warp, then the warps in order.
// Only thread 0 ends up with the sums (the other threads go on to the barrier at once).
__device__ __forceinline__ void block_reduce6(double v[6], double *smem /* [32][6] */)
{
#pragma unroll
    for (int k = 0; k < 6; ++k)
        for (int s = 16; s; s >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], s);
    int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0)
        for (int k = 0; k < 6; ++k) smem[warp * 6 + k] = v[k];
    __syncthreads();
    if (threadIdx.x != 0) return;
    int nw = blockDim.x >> 5;
    for (int k = 0; k < 6; ++k) {
        double s = 0.0;
        for (int w = 0; w < nw; ++w) s += smem[w * 6 + k];
        v[k] = s;
    }
}

// Every block sums the per-block partials in the same order -> identical totals everywhere.  The order is that of
// block_reduce6 over one partial per thread (nblocks <= blockDim): butterflies over groups of 32 blocks, then the groups
// in order.  The groups block_reduce6 would add past the last block are +0.0, which leaves a sum that started at +0.0
// unchanged, so warp 0 alone computes the totals and hands them to the block through shared memory.
__device__ __forceinline__ void grid_totals(const double *part, int nblocks, double out[6], double *smem)
{
    if (threadIdx.x < 32) {
        double s[6] = {0, 0, 0, 0, 0, 0};
        for (int b0 = 0; b0 < nblocks; b0 += 32) {
            const int b = b0 + (int)threadIdx.x;
            double v[6] = {0, 0, 0, 0, 0, 0};
            if (b < nblocks)
                for (int k = 0; k < 6; ++k) v[k] += part[(size_t)b * 8 + k];
#pragma unroll
            for (int k = 0; k < 6; ++k) {
                for (int sh = 16; sh; sh >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], sh);
                s[k] += v[k];
            }
        }
        if (threadIdx.x == 0)
            for (int k = 0; k < 6; ++k) smem[k] = s[k];
    }
    __syncthreads();
    for (int k = 0; k < 6; ++k) out[k] = smem[k];
}

constexpr int PCG_THREADS = 1024;  // one fat block per SM: grid.sync() cost grows with the block count
// Rows / entries per thread in flight.  __launch_bounds__(1024, 1) leaves 64 registers; on C3 (H100 SXM, 400 W)
// batch 2 / rows 1 spills 48 B and is fastest, batch 4 / rows 2 spills 364 B and is 5 % slower, rows 4 is 20 % slower.
constexpr int PCG_BATCH = 2;       // SpMV: column words / p gathers per row
constexpr int PCG_ROWS = 1;        // vector phases: rows per thread
__global__ void __launch_bounds__(PCG_THREADS, 1) k_pcg(Pcg q)
{
    cg::grid_group grid = cg::this_grid();
    __shared__ double smem[(PCG_THREADS / 32) * 6];
    const uint32_t R = q.R;
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
    double *partA = q.partials, *partB = q.partials + (size_t)gridDim.x * 8;
    double acc[6], tot[6];
    const bool prof = q.timing && tid == 0;
    unsigned long long tprev = prof ? pcg_timer_ns() : 0ull;
    auto lap = [&](int slot) {
        if (prof) { const unsigned long long t = pcg_timer_ns(); q.status[8 + slot] += (uint32_t)(t - tprev); tprev = t; }
    };

    // r = rhs, p = M^-1 r, rhsNorm2 = r.r, absNew = r.p; p.w carries the diagonal for the SpMV and the p update
    for (int k = 0; k < 6; ++k) acc[k] = 0.0;
    for (uint32_t i = tid; i < R; i += nth) {
        float id = q.inv_diag[i];
        float rv[3], pv[3];
        for (int c = 0; c < 3; ++c) {
            rv[c] = q.rhs[(size_t)c * R + i];
            q.r[(size_t)c * R + i] = rv[c];
            q.x[(size_t)c * R + i] = 0.0f;
            pv[c] = id * rv[c];
            acc[c] += (double)rv[c] * rv[c];
            acc[3 + c] += (double)rv[c] * pv[c];
        }
        q.p[i] = make_float4(pv[0], pv[1], pv[2], q.diag_val[i]);
    }
    block_reduce6(acc, smem);
    if (threadIdx.x == 0) for (int k = 0; k < 6; ++k) partA[(size_t)blockIdx.x * 8 + k] = acc[k];
    grid.sync();
    grid_totals(partA, gridDim.x, tot, smem);
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
    grid.sync();  // partA is rewritten below
    if (prof) tprev = pcg_timer_ns();
    while (active[0] || active[1] || active[2]) {
        // phase 1: t = A p, p.t.  Two rows per thread; per batch all column words of both rows are loaded first,
        // then all p gathers, then the products are added: the dependent chain per row is extent -> columns -> p,
        // once per PCG_BATCH entries instead of once per entry.  Per row the diagonal comes first and the edges
        // follow in storage order, and the rows of a thread are added in ascending order: bit-identical.
        for (int k = 0; k < 6; ++k) acc[k] = 0.0;
        const float lam2 = 0.1f * 0.1f;
        for (uint32_t i0 = tid; i0 < R; i0 += 2 * nth) {
            const uint32_t i1 = i0 + nth;
            const bool h1 = i1 < R;
            const uint32_t j1 = h1 ? i1 : i0;
            uint32_t a = q.csr_ptr[i0] + 1, ae = q.csr_ptr[i0 + 1];
            uint32_t b = q.csr_ptr[j1] + 1, be = h1 ? q.csr_ptr[j1 + 1] : b;
            const float4 pa = q.p[i0], pb = q.p[j1];
            float a0 = 0.0f + pa.w * pa.x, a1 = 0.0f + pa.w * pa.y, a2 = 0.0f + pa.w * pa.z;  // diagonal first
            float b0 = 0.0f + pb.w * pb.x, b1 = 0.0f + pb.w * pb.y, b2 = 0.0f + pb.w * pb.z;
            while (a < ae || b < be) {
                uint32_t ea[PCG_BATCH], eb[PCG_BATCH];
#pragma unroll
                for (int k = 0; k < PCG_BATCH; ++k) {
                    ea[k] = a + k < ae ? q.csr_enc[a + k] : 0u;
                    eb[k] = b + k < be ? q.csr_enc[b + k] : 0u;
                }
                float4 va[PCG_BATCH], vb[PCG_BATCH];
#pragma unroll
                for (int k = 0; k < PCG_BATCH; ++k) {
                    va[k] = a + k < ae ? q.p[ea[k] & 0x7FFFFFFFu] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
                    vb[k] = b + k < be ? q.p[eb[k] & 0x7FFFFFFFu] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
                }
#pragma unroll
                for (int k = 0; k < PCG_BATCH; ++k) {
                    if (a + k < ae) { const float w = (ea[k] >> 31) ? -1.0f : -lam2; a0 += w * va[k].x; a1 += w * va[k].y; a2 += w * va[k].z; }
                    if (b + k < be) { const float w = (eb[k] >> 31) ? -1.0f : -lam2; b0 += w * vb[k].x; b1 += w * vb[k].y; b2 += w * vb[k].z; }
                }
                a += PCG_BATCH;
                b += PCG_BATCH;
            }
            q.t[i0] = a0; q.t[(size_t)R + i0] = a1; q.t[2 * (size_t)R + i0] = a2;
            acc[0] += (double)pa.x * a0; acc[1] += (double)pa.y * a1; acc[2] += (double)pa.z * a2;
            if (h1) {
                q.t[i1] = b0; q.t[(size_t)R + i1] = b1; q.t[2 * (size_t)R + i1] = b2;
                acc[0] += (double)pb.x * b0; acc[1] += (double)pb.y * b1; acc[2] += (double)pb.z * b2;
            }
        }
        block_reduce6(acc, smem);
        if (threadIdx.x == 0) for (int k = 0; k < 6; ++k) partA[(size_t)blockIdx.x * 8 + k] = acc[k];
        lap(0);
        grid.sync();
        grid_totals(partA, gridDim.x, tot, smem);
        lap(1);
        float alpha[3];
        bool moved[3];   // channels whose x takes this iteration's step alpha p (applied in phase 3, where p is loaded anyway)
        for (int c = 0; c < 3; ++c) {
            alpha[c] = active[c] ? absNew[c] / (float)tot[c] : 0.0f;
            moved[c] = active[c];
        }

        // phase 2: r -= a t, |r|^2, r.z (PCG_ROWS rows per thread in flight, loads first, rows added in ascending order)
        for (int k = 0; k < 6; ++k) acc[k] = 0.0;
        for (uint32_t i = tid; i < R; i += PCG_ROWS * nth) {
            float id[PCG_ROWS], rr[PCG_ROWS][3], tt[PCG_ROWS][3];
#pragma unroll
            for (int u = 0; u < PCG_ROWS; ++u) {
                const uint32_t j = i + u * nth;
                id[u] = 0.0f;
#pragma unroll
                for (int c = 0; c < 3; ++c) { rr[u][c] = 0.0f; tt[u][c] = 0.0f; }
                if (j >= R) continue;
                id[u] = q.inv_diag[j];
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    if (active[c]) { rr[u][c] = q.r[(size_t)c * R + j]; tt[u][c] = q.t[(size_t)c * R + j]; }
            }
#pragma unroll
            for (int u = 0; u < PCG_ROWS; ++u) {
                const uint32_t j = i + u * nth;
                if (j >= R) continue;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    if (!active[c]) continue;
                    const float rv = rr[u][c] - alpha[c] * tt[u][c];
                    q.r[(size_t)c * R + j] = rv;
                    acc[c] += (double)rv * rv;
                    acc[3 + c] += (double)rv * (id[u] * rv);
                }
            }
        }
        block_reduce6(acc, smem);
        if (threadIdx.x == 0) for (int k = 0; k < 6; ++k) partB[(size_t)blockIdx.x * 8 + k] = acc[k];
        lap(2);
        grid.sync();
        grid_totals(partB, gridDim.x, tot, smem);
        lap(3);
        float beta[3] = {0.0f, 0.0f, 0.0f};
        bool upd[3];
        for (int c = 0; c < 3; ++c) {
            upd[c] = false;
            if (!active[c]) continue;
            resNorm2[c] = (float)tot[c];
            if (resNorm2[c] < threshold[c]) { active[c] = false; continue; }  // break before ++i
            float absOld = absNew[c];
            absNew[c] = (float)tot[3 + c];
            beta[c] = absNew[c] / absOld;
            upd[c] = true;
            if (++iters[c] >= q.max_iters) active[c] = false;  // while (i < maxIters)
        }
        // phase 3: x += a p with the p of this iteration, then p = z + beta p (PCG_ROWS rows per thread in flight).
        // Runs in every iteration: some channel was active in phase 2, or the loop would have ended.
        const bool pu = upd[0] || upd[1] || upd[2];
        for (uint32_t i = tid; i < R; i += PCG_ROWS * nth) {
            float4 pv[PCG_ROWS];
            float xx[PCG_ROWS][3], rr[PCG_ROWS][3];
#pragma unroll
            for (int u = 0; u < PCG_ROWS; ++u) {
                const uint32_t j = i + u * nth;
                pv[u] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
#pragma unroll
                for (int c = 0; c < 3; ++c) { xx[u][c] = 0.0f; rr[u][c] = 0.0f; }
                if (j >= R) continue;
                pv[u] = q.p[j];
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    if (moved[c]) xx[u][c] = q.x[(size_t)c * R + j];
                    if (upd[c]) rr[u][c] = q.r[(size_t)c * R + j];
                }
            }
#pragma unroll
            for (int u = 0; u < PCG_ROWS; ++u) {
                const uint32_t j = i + u * nth;
                if (j >= R) continue;
                if (moved[0]) q.x[j] = xx[u][0] + alpha[0] * pv[u].x;
                if (moved[1]) q.x[(size_t)R + j] = xx[u][1] + alpha[1] * pv[u].y;
                if (moved[2]) q.x[2 * (size_t)R + j] = xx[u][2] + alpha[2] * pv[u].z;
                if (!pu) continue;
                const float d = pv[u].w;
                const float id = d != 0.0f ? 1.0f / d : 1.0f;   // = inv_diag (k_matrix): same expression, same bits
                if (upd[0]) pv[u].x = id * rr[u][0] + beta[0] * pv[u].x;
                if (upd[1]) pv[u].y = id * rr[u][1] + beta[1] * pv[u].y;
                if (upd[2]) pv[u].z = id * rr[u][2] + beta[2] * pv[u].z;
                q.p[j] = pv[u];
            }
        }
        lap(4);
        ++loops;
        grid.sync();
        lap(5);
    }
    // x -= mean(x)  (:277)
    for (int k = 0; k < 6; ++k) acc[k] = 0.0;
    for (uint32_t i = tid; i < R; i += nth)
        for (int c = 0; c < 3; ++c) acc[c] += (double)q.x[(size_t)c * R + i];
    block_reduce6(acc, smem);
    if (threadIdx.x == 0) for (int k = 0; k < 6; ++k) partA[(size_t)blockIdx.x * 8 + k] = acc[k];
    grid.sync();
    grid_totals(partA, gridDim.x, tot, smem);
    float mean[3];
    for (int c = 0; c < 3; ++c) mean[c] = R ? (float)(tot[c] / (double)R) : 0.0f;
    for (uint32_t i = tid; i < R; i += nth)
        for (int c = 0; c < 3; ++c) q.x[(size_t)c * R + i] -= mean[c];
    if (tid == 0) {
        for (int c = 0; c < 3; ++c) {
            q.status[c] = iters[c];
            float err = rhsNorm2[c] != 0.0f ? sqrtf(resNorm2[c] / rhsNorm2[c]) : 0.0f;
            q.status[3 + c] = __float_as_uint(err);
        }
        q.status[6] = loops;
    }
}

}  // namespace

int seam_run(b2tex_ctx *c, b2tex_seam_info *info, bool solve)
{
    invalidate(c, SEAM_SYSTEM);
    if (!c->Vn || !c->K) { set_error("seam leveling: mesh, vertex rings, labels and views must be set"); return B2TEX_ERR_ARG; }
    B2_TRY(require(c, MESH | PIXELS | RINGS | LABELS, "seam leveling"));
    cudaStream_t s = c->stream;
    // only the camera block and the rgb images are needed here (no gradient image)
    B2_TRY(prepare_images(c, (c->valid & IMAGES) ? c->prepared_data_term : 0));
    const uint32_t Vn = c->Vn;
    std::unique_ptr<ScopedTimer> tm_asm(new ScopedTimer(c, "seam_assembly"));
    DevBuf<uint32_t> &cnt = c->s_cnt32, &row_vertex = c->s_row_vertex;
    B2_TRY(cnt.alloc((size_t)Vn + 1));
    B2_TRY(cnt.zero(s));
    B2_TRY(c->s_limits.alloc(1));
    B2_TRY(c->s_limits.zero(s));
    uint32_t *limit_flags = c->s_limits.p;   // bit 0: MAXL labels on a vertex, bit 1: > 16 faces on an edge
    B2_TRY(c->row_ptr.alloc((size_t)Vn + 1));
    const uint32_t vb = (Vn + 127) / 128;
    B2_LAUNCH k_vertex_labels<false><<<vb, 128, 0, s>>>(Vn, c->vf_ptr.p, c->vf_idx.p, c->labels.p, cnt.p, nullptr, nullptr, nullptr,
                                              limit_flags);
    B2_KERNEL_CHECK();
    B2_TRY(cub_exclusive_sum_u32(c, cnt.p, c->row_ptr.p, (size_t)Vn + 1));
    uint32_t R = 0;
    B2_CUDA(cudaMemcpyAsync(&R, c->row_ptr.p + Vn, 4, cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaStreamSynchronize(s));
    c->R = R;
    B2_TRY(c->row_label.alloc(R));
    B2_TRY(row_vertex.alloc(R));
    B2_LAUNCH k_vertex_labels<true><<<vb, 128, 0, s>>>(Vn, c->vf_ptr.p, c->vf_idx.p, c->labels.p, nullptr, c->row_ptr.p,
                                             c->row_label.p, row_vertex.p, limit_flags);
    B2_KERNEL_CHECK();

    SeamMesh m{c->verts.p, c->faces.p, c->vf_ptr.p, c->vf_idx.p, c->vv_ptr.p, c->vv_idx.p, c->labels.p,
               c->row_ptr.p, c->row_label.p, c->views_dev.p};
    B2_TRY(c->arow_ptr.alloc((size_t)Vn + 1));
    B2_TRY(cnt.zero(s));
    B2_LAUNCH k_arows<false><<<vb, 128, 0, s>>>(Vn, m, cnt.p, nullptr, nullptr, nullptr, limit_flags);
    B2_KERNEL_CHECK();
    B2_TRY(cub_exclusive_sum_u32(c, cnt.p, c->arow_ptr.p, (size_t)Vn + 1));
    uint32_t A = 0;
    B2_CUDA(cudaMemcpyAsync(&A, c->arow_ptr.p + Vn, 4, cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaStreamSynchronize(s));
    c->A_rows = A;
    B2_TRY(c->arow_rows.alloc(2 * (size_t)A));
    B2_TRY(c->arow_b.alloc(3 * (size_t)A));
    B2_LAUNCH k_arows<true><<<vb, 128, 0, s>>>(Vn, m, nullptr, c->arow_ptr.p, c->arow_rows.p, c->arow_b.p, limit_flags);
    B2_KERNEL_CHECK();

    DevBuf<uint32_t> &rcnt = c->s_rcnt;
    B2_TRY(rcnt.alloc((size_t)R + 1));
    B2_TRY(rcnt.zero(s));
    B2_TRY(c->csr_ptr.alloc((size_t)R + 1));
    const uint32_t rb = (R + 127) / 128;
    if (R)
        B2_LAUNCH k_matrix<false><<<rb, 128, 0, s>>>(R, m, row_vertex.p, c->arow_ptr.p, c->arow_rows.p, c->arow_b.p, rcnt.p,
                                           nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
    B2_KERNEL_CHECK();
    B2_TRY(cub_exclusive_sum_u32(c, rcnt.p, c->csr_ptr.p, (size_t)R + 1));
    uint32_t nnzL = 0, limits = 0;
    B2_CUDA(cudaMemcpyAsync(&nnzL, c->csr_ptr.p + R, 4, cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaMemcpyAsync(&limits, limit_flags, 4, cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaStreamSynchronize(s));
    if (limits) {
        set_error("global seam leveling: %s%s", (limits & 1u) ? "a vertex carries more than 64 different labels; " : "",
                  (limits & 2u) ? "an edge has more than 16 incident faces" : "");
        return B2TEX_ERR_LIMITS;
    }
    c->nnz_L = nnzL;
    B2_TRY(c->csr_col.alloc(nnzL));
    B2_TRY(c->csr_val.alloc(nnzL));
    B2_TRY(c->csr_enc.alloc(nnzL));
    B2_TRY(c->seam_dval.alloc(R));
    B2_TRY(c->seam_diag.alloc(R));
    B2_TRY(c->seam_rhs.alloc(3 * (size_t)R));
    B2_TRY(c->seam_x.alloc(3 * (size_t)R));
    B2_TRY(c->seam_r.alloc(3 * (size_t)R));
    B2_TRY(c->seam_t.alloc(3 * (size_t)R));
    B2_TRY(c->seam_p.alloc(R));
    if (R)
        B2_LAUNCH k_matrix<true><<<rb, 128, 0, s>>>(R, m, row_vertex.p, c->arow_ptr.p, c->arow_rows.p, c->arow_b.p, nullptr,
                                          c->csr_ptr.p, c->csr_col.p, c->csr_val.p, c->seam_diag.p, c->seam_rhs.p, c->csr_enc.p,
                                          c->seam_dval.p);
    B2_KERNEL_CHECK();
    mark_valid(c, SEAM_SYSTEM);

    // Gamma rows = sum over rows of Gamma neighbours / 2
    info->num_rows = R;
    info->num_a_rows = A;
    info->nnz_full = nnzL;
    info->num_gamma_rows = (uint32_t)((nnzL - R - 2ull * A) / 2ull);
    for (int ch = 0; ch < 3; ++ch) { info->iterations[ch] = 0; info->residual[ch] = 0.0f; }
    info->cg_launch_iterations = 0;
    info->cg_ms = 0.0f;

    tm_asm.reset();
    B2_TRY(c->seam_status.alloc(16));
    B2_TRY(c->seam_status.zero(s));
    if (R && solve) {   // solve == false: assembly only, the multi-GPU solver (seam_mg.cu) takes over
        int per_sm = 0;
        B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pcg, PCG_THREADS, 0));
        if (per_sm < 1) { set_error("k_pcg cannot be resident"); return B2TEX_ERR_CUDA; }
        int grid = c->num_sms * per_sm;
        int need = (int)((R + PCG_THREADS - 1) / PCG_THREADS);
        if (grid > need) grid = std::max(1, need);
        grid = std::min(grid, PCG_THREADS);   // grid_totals: at most one block partial per thread
        B2_TRY(c->seam_partials.alloc(2 * (size_t)grid * 8));
        Pcg q{R, c->csr_ptr.p, c->csr_enc.p, c->seam_dval.p, c->seam_diag.p, c->seam_rhs.p, c->seam_x.p,
              c->seam_r.p, c->seam_t.p, c->seam_p.p, c->seam_partials.p, c->seam_status.p, 1000u, 0.0001f};
        static const bool seam_timing = getenv("B2TEX_SEAM_TIMING") != nullptr;
        q.timing = seam_timing ? 1u : 0u;
        void *args[] = {&q};
        cudaEvent_t e0, e1;
        B2_CUDA(cudaEventCreate(&e0));
        B2_CUDA(cudaEventCreate(&e1));
        B2_CUDA(cudaEventRecord(e0, s));
        count_launch();
        B2_CUDA(cudaLaunchCooperativeKernel((void *)k_pcg, dim3(grid), dim3(PCG_THREADS), args, 0, s));
        B2_CUDA(cudaEventRecord(e1, s));
        uint32_t st[16];
        B2_CUDA(cudaMemcpyAsync(st, c->seam_status.p, sizeof(st), cudaMemcpyDeviceToHost, s));
        B2_CUDA(cudaStreamSynchronize(s));
        float ms = 0.0f;
        cudaEventElapsedTime(&ms, e0, e1);
        cudaEventDestroy(e0);
        cudaEventDestroy(e1);
        if (seam_timing)
            fprintf(stderr, "k_pcg: %u iterations, grid %d, %.3f ms, block 0 [us]: spmv %.0f barrier_a %.0f update %.0f barrier_b %.0f "
                    "p %.0f loop_barrier %.0f\n", st[6], grid, ms, st[8] / 1e3, st[9] / 1e3, st[10] / 1e3, st[11] / 1e3, st[12] / 1e3,
                    st[13] / 1e3);
        for (int ch = 0; ch < 3; ++ch) {
            info->iterations[ch] = st[ch];
            memcpy(&info->residual[ch], &st[3 + ch], 4);
        }
        info->cg_launch_iterations = st[6];
        info->cg_ms = ms;
    }
    if (solve) mark_valid(c, SEAM);
    return B2TEX_OK;
}

}  // namespace b2
