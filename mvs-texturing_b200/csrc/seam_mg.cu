// seam_mg.cu -- K9': the global seam leveling solve across GPUs, ONE kernel per GPU doing compute + exchange.
//
// Replaces the replicated k_pcg (seam.cu) when the job runs on several GPUs (one process per GPU): the rows of
// Lhs x = Rhs (global_seam_leveling.cpp:245-277) are split into contiguous ranges, one per rank.  Every rank runs the
// same persistent Jacobi-PCG as k_pcg on ITS rows and, inside the kernel, exchanges with its peers through peer-mapped
// memory (cudaIpc handles, NVLink / NVSwitch stores) instead of returning to the host for NCCL:
//   * halo of the search direction: a rank's SpMV reads p of a few rows it does not own (0.4 % of the rows at 2 ranks,
//     2 % at 8 on the C3 system: the Laplacian couples a vertex only to its 1-ring).  It keeps its OWN copy of p for those
//     rows and updates it itself: the owner stores z = M^-1 r of its halo rows into the readers' z arrays right after the
//     residual update -- BEFORE the all-reduce that yields beta -- and every reader then forms p = z + beta p for its
//     imported rows with the same two roundings as the owner.  The exchange therefore rides on the barrier of the
//     all-reduce that CG needs anyway; there is no third cross-GPU barrier per iteration;
//   * dot products: two all-reduces per iteration (p.t; |r|^2 and r.z).  Every block leaves its fp64 partial sums in a
//     table and takes a ticket; the LAST block of the rank adds the table in block order and stores the rank's sums into
//     slot [parity][rank] of every peer as twelve 8-byte words {32 bits of payload, epoch}: payload and flag travel in one
//     store, so neither side needs a system-scope fence (the "LL" protocol of collective libraries); all blocks of all
//     ranks poll the P x 12 words of the epoch and add the P slots in rank order -> bit-identical scalars on every GPU.
//     This one step is reduction, cross-GPU barrier and grid-wide barrier at once (no cooperative-groups grid.sync in the
//     loop).  The halo entries of z are self-validating in the same way: the unused fourth component of the float4
//     carries the epoch, the reader polls the entry itself;
//   * one device-local barrier per iteration (ticket counter) between the update of p and the next SpMV.
// Results are deterministic for a given rank count and grid; they differ from the single-GPU kernel only by the
// summation order of the reductions (per block, per rank, then across ranks).
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"

namespace b2 {

constexpr int MG_MAX_RANKS = 8;

// Layout of the peer-visible block every rank allocates (and exports through one cudaIpc handle):
//   float4 p[R] | float4 z[R] | float x[3][R] | uint2 ll[2][MG_MAX_RANKS][12] | uint32 flag[MG_MAX_RANKS] (padded to 64 B)
// p is only written by the owner of the block; z (halo rows, w = epoch tag), x (final all-gather) and ll (all-reduce slots:
// {half of a double, epoch} per word) are written by peers.
constexpr int MG_LL_WORDS = 12;   // six doubles as twelve self-validating 8-byte words
struct MgBlock {
    float4 *p, *z;
    float *x;
    uint2 *ll;
    uint32_t *flag;
};
// every section starts on a 64-byte boundary (R may be odd: 12 R bytes would leave the doubles misaligned)
__host__ __device__ inline size_t mg_align64(size_t n) { return (n + 63) & ~(size_t)63; }
__host__ __device__ inline size_t mg_block_bytes(uint32_t R)
{
    return 2 * mg_align64((size_t)R * 16) + mg_align64((size_t)R * 12) + mg_align64(2 * MG_MAX_RANKS * MG_LL_WORDS * sizeof(uint2)) + 64;
}
__host__ __device__ inline MgBlock mg_carve(void *base, uint32_t R)
{
    MgBlock b;
    char *c = (char *)base;
    b.p = (float4 *)c; c += mg_align64((size_t)R * 16);
    b.z = (float4 *)c; c += mg_align64((size_t)R * 16);
    b.x = (float *)c; c += mg_align64((size_t)R * 12);
    b.ll = (uint2 *)c; c += mg_align64(2 * MG_MAX_RANKS * MG_LL_WORDS * sizeof(uint2));
    b.flag = (uint32_t *)c;
    return b;
}

struct PcgMg {
    uint32_t R, r0, r1;          // system size, own row range [r0, r1)
    uint32_t rank, nranks;
    const uint32_t *csr_ptr, *csr_enc;
    const float *diag_val, *inv_diag, *rhs;   // replicated assembly (k_matrix), indexed by global row
    float *r, *t;                // [3][R] local scratch (own rows used)
    const uint8_t *dest;         // [R] for own rows: bit k = rank k reads this row's entry of p (halo destination mask)
    const uint32_t *imp;         // rows of other ranks whose entry of p this rank's SpMV reads (halo imports)
    const uint32_t *n_imp;       // their number (device side: written by k_pcg_mg_imports)
    double *blockpart;           // [grid][8] per-block partials of this rank
    uint32_t *status;            // [0..2] iterations, [3..5] residual bits, [6] loops, [7] barrier timeouts, [8] epoch,
                                 // [10] tickets of the all-reduces, [11] tickets of the device-local barrier,
                                 // [16..21] ns block 0 spent in SpMV / all-reduce A / update / all-reduce B / p / local barrier
    uint32_t timing;             // diagnostic (B2TEX_SEAM_TIMING): fill status[16..21]
    void *peer[MG_MAX_RANKS];    // base pointers of every rank's MgBlock (peer[rank] = own)
    uint32_t max_iters;
    float tol;
    uint32_t epoch0;             // barrier epochs used so far (blocks are reused across solves)
    unsigned long long spin_limit;
};

namespace {

__device__ __forceinline__ void st_release_sys(uint32_t *p, uint32_t v)
{
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t *p)
{
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// 8- and 16-byte accesses that are performed as ONE transaction and never cached in L1 (payload and tag arrive together)
__device__ __forceinline__ void st_volatile_v2(uint2 *p, uint32_t a, uint32_t b)
{
    asm volatile("st.volatile.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ uint2 ld_volatile_v2(const uint2 *p)
{
    uint2 v;
    asm volatile("ld.volatile.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_volatile_v4(float4 *p, float a, float b, float c, uint32_t tag)
{
    asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(__float_as_uint(a)), "r"(__float_as_uint(b)),
                 "r"(__float_as_uint(c)), "r"(tag) : "memory");
}
__device__ __forceinline__ uint4 ld_volatile_v4(const float4 *p)
{
    uint4 v;
    asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long mg_timer_ns()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t *p)
{
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// Sum of six doubles over the block, in a fixed order: shuffles inside every warp, one row per warp in shared memory,
// then the first warp adds the rows (lane = warp) by shuffles again.  Only thread 0 ends up with the sums.
__device__ __forceinline__ void mg_block_reduce6(double v[6], double *smem)
{
    for (int k = 0; k < 6; ++k)
        for (int s = 16; s; s >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], s);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0)
        for (int k = 0; k < 6; ++k) smem[warp * 6 + k] = v[k];
    __syncthreads();
    if (warp == 0) {
        const int nw = blockDim.x >> 5;
        for (int k = 0; k < 6; ++k) {
            double s = lane < nw ? smem[lane * 6 + k] : 0.0;
            for (int d = 16; d; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
            v[k] = s;
        }
    }
}

// All-reduce of six partial sums across all blocks of all ranks = grid-wide barrier + cross-GPU barrier, in one step.
// `seq` counts the calls of this solve (1, 2, ...): the ticket that completes call `seq` is seq * gridDim.x.  `remote`:
// this rank stored ordinary data into peer memory since the previous call (the final all-gather of x): those stores are
// fenced at system scope by one thread per block, after the block's own barrier, before the ticket, and once more before
// the words go out; then everything any thread of any rank stored before its call is visible to every thread of every
// rank after it.  Inside the iteration nothing needs that: the halo of z validates itself.
__device__ __forceinline__ bool mg_allreduce6(const PcgMg &q, double acc[6], double *smem, uint32_t *s_last, int parity,
                                              uint32_t epoch, uint32_t seq, bool remote, bool alive, double tot[6])
{
    // after a timeout (a peer or a block is gone) nobody waits any more; `alive` is uniform within a block, and no
    // construct below needs it to be uniform across blocks (tickets and polls all time out by themselves)
    if (!alive) { for (int k = 0; k < 6; ++k) tot[k] = 0.0; return false; }
    mg_block_reduce6(acc, smem);
    if (threadIdx.x == 0) {
        for (int k = 0; k < 6; ++k) q.blockpart[(size_t)blockIdx.x * 8 + k] = acc[k];
        if (remote) __threadfence_system(); else __threadfence();
        const uint32_t ticket = atomicAdd(q.status + 10, 1u);
        *s_last = (ticket + 1u == seq * gridDim.x) ? 1u : 0u;
    }
    __syncthreads();
    if (*s_last) {   // the last block of this rank: every other block's partials and stores are behind its ticket
        __threadfence();
        double v[6] = {0, 0, 0, 0, 0, 0};
        for (uint32_t b = threadIdx.x; b < gridDim.x; b += blockDim.x)
            for (int k = 0; k < 6; ++k) v[k] += __ldcg(q.blockpart + (size_t)b * 8 + k);
        mg_block_reduce6(v, smem);
        __syncthreads();
        if (threadIdx.x == 0) for (int k = 0; k < 6; ++k) smem[k] = v[k];
        __syncthreads();
        if (threadIdx.x < q.nranks * MG_LL_WORDS) {   // one 8-byte word {half of a sum, epoch} per thread
            const uint32_t k = threadIdx.x / MG_LL_WORDS, hw = threadIdx.x % MG_LL_WORDS;
            const unsigned long long bits = (unsigned long long)__double_as_longlong(smem[hw >> 1]);
            if (remote) __threadfence_system();   // the final all-gather of x: ordinary stores before the words that announce them
            st_volatile_v2(mg_carve(q.peer[k], q.R).ll + ((size_t)parity * MG_MAX_RANKS + q.rank) * MG_LL_WORDS + hw,
                           (uint32_t)(bits >> (32 * (hw & 1u))), epoch);
        }
    }
    // every block collects the words of every rank (its own included): P x 12 pollers, payload and tag in one load
    uint32_t *halves = reinterpret_cast<uint32_t *>(smem);   // [P][12]; smem is free again after the block reduction
    __syncthreads();
    if (threadIdx.x < q.nranks * MG_LL_WORDS) {
        const uint2 *w = mg_carve(q.peer[q.rank], q.R).ll + (size_t)parity * MG_MAX_RANKS * MG_LL_WORDS +
                         (size_t)(threadIdx.x / MG_LL_WORDS) * MG_LL_WORDS + threadIdx.x % MG_LL_WORDS;
        unsigned long long spins = 0;
        uint2 got = ld_volatile_v2(w);
        while (got.y != epoch) {
            if (++spins > 64) __nanosleep(20);   // the words normally arrive within a few microseconds: poll hard first
            if (spins > q.spin_limit) { atomicAdd(q.status + 7, 1u); break; }
            got = ld_volatile_v2(w);
        }
        halves[threadIdx.x] = got.x;
    }
    __syncthreads();
    if (threadIdx.x == 0) s_last[1] = __ldcg(q.status + 7);   // one verdict per block
    for (int k = 0; k < 6; ++k) {
        double sum = 0.0;
        for (uint32_t r = 0; r < q.nranks; ++r) {   // rank order: identical on every GPU
            const unsigned long long bits = (unsigned long long)halves[r * MG_LL_WORDS + 2 * k] |
                                            ((unsigned long long)halves[r * MG_LL_WORDS + 2 * k + 1] << 32);
            sum += __longlong_as_double((long long)bits);
        }
        tot[k] = sum;
    }
    __syncthreads();
    return s_last[1] == 0u;
}

// device-local barrier of the persistent grid (ticket counter; a timeout instead of a hang if a block went away)
__device__ __forceinline__ bool mg_local_sync(const PcgMg &q, uint32_t *s_last, uint32_t seq, bool alive)
{
    if (!alive) return false;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(q.status + 11, 1u);
        const uint32_t target = seq * gridDim.x;
        unsigned long long spins = 0;
        while ((int32_t)(ld_acquire_gpu(q.status + 11) - target) < 0) {
            __nanosleep(20);
            if (++spins > q.spin_limit) { atomicAdd(q.status + 7, 1u); break; }
        }
        s_last[1] = __ldcg(q.status + 7);
    }
    __syncthreads();
    return s_last[1] == 0u;
}

// z = M^-1 r of one own row goes to the ranks that read this row's entry of p
__device__ __forceinline__ void mg_push_z(const PcgMg &q, uint32_t i, float a, float b, float c, uint32_t tag)
{
    for (uint32_t mk = q.dest[i]; mk; mk &= mk - 1u) {
        const uint32_t k = (uint32_t)__ffs((int)mk) - 1u;
        st_volatile_v4(mg_carve(q.peer[k], q.R).z + i, a, b, c, tag);   // one 16-byte store: values and tag arrive together
    }
}

// owner of a row: rank k owns [R k / P, R (k + 1) / P)
__device__ __forceinline__ uint32_t mg_owner(uint32_t row, uint32_t R, uint32_t nranks)
{
    uint32_t k = (uint32_t)(((uint64_t)row * nranks) / R);
    while (k + 1 < nranks && row >= (uint32_t)((uint64_t)R * (k + 1) / nranks)) ++k;
    while (k > 0 && row < (uint32_t)((uint64_t)R * k / nranks)) --k;
    return k;
}

}  // namespace

// destination mask of every own row: the ranks whose row ranges hold a row with this row among its columns (the matrix is
// symmetric: those are the owners of this row's own columns); the same pass marks the columns this rank imports
__global__ void __launch_bounds__(256) k_pcg_mg_dest(uint32_t R, uint32_t r0, uint32_t r1, uint32_t rank, uint32_t nranks,
                                                     const uint32_t *__restrict__ csr_ptr, const uint32_t *__restrict__ csr_enc,
                                                     uint8_t *dest, uint8_t *imp_mark)
{
    const uint32_t i = r0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= r1) return;
    uint32_t mask = 0;
    for (uint32_t e = csr_ptr[i] + 1; e < csr_ptr[i + 1]; ++e) {
        const uint32_t col = csr_enc[e] & 0x7FFFFFFFu;
        const uint32_t k = mg_owner(col, R, nranks);
        if (k != rank) { mask |= 1u << k; imp_mark[col] = 1; }
    }
    dest[i] = (uint8_t)mask;
}
// the marked rows, in any order
__global__ void __launch_bounds__(256) k_pcg_mg_imports(uint32_t R, const uint8_t *__restrict__ imp_mark, uint32_t *imp, uint32_t *n_imp)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < R && imp_mark[i]) imp[atomicAdd(n_imp, 1u)] = i;
}

constexpr int MG_THREADS = 1024;
__global__ void __launch_bounds__(MG_THREADS, 1) k_pcg_mg(PcgMg q)
{
    __shared__ double smem[(MG_THREADS / 32) * 6 + 1];
    uint32_t *s_last = reinterpret_cast<uint32_t *>(smem + (MG_THREADS / 32) * 6);   // [0] "last block of the rank", [1] failure verdict
    const uint32_t R = q.R;
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
    const MgBlock own = mg_carve(q.peer[q.rank], R);
    const uint32_t n_imp = *q.n_imp;
    double acc[6], tot[6];
    uint32_t epoch = q.epoch0, seq = 0, lseq = 0;
    int parity = 0;
    bool alive = true;
    const bool prof = q.timing && tid == 0;
    unsigned long long tprev = prof ? mg_timer_ns() : 0ull;
    auto lap = [&](int slot) {
        if (prof) { const unsigned long long t = mg_timer_ns(); q.status[16 + slot] += (uint32_t)(t - tprev); tprev = t; }
    };

    // r = rhs, p = M^-1 r on the own rows AND on the imported rows (the assembly is replicated: no exchange needed)
    for (int k = 0; k < 6; ++k) acc[k] = 0.0;
    for (uint32_t i = q.r0 + tid; i < q.r1; i += nth) {
        const float id = q.inv_diag[i];
        float pv[3];
        for (int c = 0; c < 3; ++c) {
            const float rv = q.rhs[(size_t)c * R + i];
            q.r[(size_t)c * R + i] = rv;
            own.x[(size_t)c * R + i] = 0.0f;
            pv[c] = id * rv;
            acc[c] += (double)rv * rv;
            acc[3 + c] += (double)rv * pv[c];
        }
        own.p[i] = make_float4(pv[0], pv[1], pv[2], 0.0f);
    }
    for (uint32_t j = tid; j < n_imp; j += nth) {
        const uint32_t i = q.imp[j];
        const float id = q.inv_diag[i];
        own.p[i] = make_float4(id * q.rhs[i], id * q.rhs[(size_t)R + i], id * q.rhs[2 * (size_t)R + i], 0.0f);
    }
    alive = mg_allreduce6(q, acc, smem, s_last, parity, ++epoch, ++seq, false, alive, tot); parity ^= 1;
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
    const float lam2 = 0.1f * 0.1f;
    while (alive && (active[0] || active[1] || active[2])) {
        // phase 1: t = A p on the own rows (own entries and the imported halo entries are local), p.t; two rows in flight
        for (int k = 0; k < 6; ++k) acc[k] = 0.0;
        for (uint32_t i0 = q.r0 + tid; i0 < q.r1; i0 += 2 * nth) {
            const uint32_t i1 = i0 + nth;
            const bool h1 = i1 < q.r1;
            uint32_t a = q.csr_ptr[i0] + 1, ae = q.csr_ptr[i0 + 1];
            uint32_t b = h1 ? q.csr_ptr[i1] + 1 : 0u, be = h1 ? q.csr_ptr[i1 + 1] : 0u;
            const float4 pa = own.p[i0];
            const float4 pb = h1 ? own.p[i1] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
            const float da = q.diag_val[i0], db = h1 ? q.diag_val[i1] : 0.0f;
            float a0 = 0.0f + da * pa.x, a1 = 0.0f + da * pa.y, a2 = 0.0f + da * pa.z;
            float b0 = 0.0f + db * pb.x, b1 = 0.0f + db * pb.y, b2 = 0.0f + db * pb.z;
            while (a < ae || b < be) {
                uint32_t ea = 0, eb = 0;
                if (a < ae) ea = q.csr_enc[a];
                if (b < be) eb = q.csr_enc[b];
                float4 va = make_float4(0.0f, 0.0f, 0.0f, 0.0f), vb = va;
                if (a < ae) va = own.p[ea & 0x7FFFFFFFu];
                if (b < be) vb = own.p[eb & 0x7FFFFFFFu];
                if (a < ae) { const float w = (ea >> 31) ? -1.0f : -lam2; a0 += w * va.x; a1 += w * va.y; a2 += w * va.z; ++a; }
                if (b < be) { const float w = (eb >> 31) ? -1.0f : -lam2; b0 += w * vb.x; b1 += w * vb.y; b2 += w * vb.z; ++b; }
            }
            q.t[i0] = a0; q.t[(size_t)R + i0] = a1; q.t[2 * (size_t)R + i0] = a2;
            acc[0] += (double)pa.x * a0; acc[1] += (double)pa.y * a1; acc[2] += (double)pa.z * a2;
            if (h1) {
                q.t[i1] = b0; q.t[(size_t)R + i1] = b1; q.t[2 * (size_t)R + i1] = b2;
                acc[0] += (double)pb.x * b0; acc[1] += (double)pb.y * b1; acc[2] += (double)pb.z * b2;
            }
        }
        lap(0);
        alive = mg_allreduce6(q, acc, smem, s_last, parity, ++epoch, ++seq, false, alive, tot); parity ^= 1;
        lap(1);
        float alpha[3];
        for (int c = 0; c < 3; ++c) alpha[c] = active[c] ? absNew[c] / (float)tot[c] : 0.0f;

        // phase 2: x += a p, r -= a t, |r|^2, r.z; z = M^-1 r of the halo rows goes to the ranks that read them
        for (int k = 0; k < 6; ++k) acc[k] = 0.0;
        for (uint32_t i = q.r0 + tid; i < q.r1; i += nth) {
            const float4 pi = own.p[i];
            const float pv[3] = {pi.x, pi.y, pi.z};
            const float id = q.inv_diag[i];
            float xv[3], rv0[3], tv[3], zv[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll
            for (int c = 0; c < 3; ++c) { const size_t o = (size_t)c * R + i; xv[c] = own.x[o]; rv0[c] = q.r[o]; tv[c] = q.t[o]; }
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                if (!active[c]) continue;
                const size_t o = (size_t)c * R + i;
                own.x[o] = xv[c] + alpha[c] * pv[c];
                const float rv = rv0[c] - alpha[c] * tv[c];
                q.r[o] = rv;
                zv[c] = id * rv;
                acc[c] += (double)rv * rv;
                acc[3 + c] += (double)rv * zv[c];
            }
            if (q.dest[i]) mg_push_z(q, i, zv[0], zv[1], zv[2], epoch + 1u);   // tag = the epoch of the all-reduce that follows
        }
        lap(2);
        alive = mg_allreduce6(q, acc, smem, s_last, parity, ++epoch, ++seq, false, alive, tot); parity ^= 1;
        lap(3);
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
        // phase 3: p = z + beta p on the own rows and, from the z the owners pushed, on the imported rows
        if (upd[0] || upd[1] || upd[2]) {
            for (uint32_t i = q.r0 + tid; i < q.r1; i += nth) {
                float4 pi = own.p[i];
                const float id = q.inv_diag[i];
                const float r0v = q.r[i], r1v = q.r[(size_t)R + i], r2v = q.r[2 * (size_t)R + i];
                if (upd[0]) pi.x = id * r0v + beta[0] * pi.x;
                if (upd[1]) pi.y = id * r1v + beta[1] * pi.y;
                if (upd[2]) pi.z = id * r2v + beta[2] * pi.z;
                own.p[i] = pi;
            }
            for (uint32_t j = tid; j < n_imp; j += nth) {
                const uint32_t i = q.imp[j];
                float4 pi = own.p[i];
                uint4 zi = ld_volatile_v4(own.z + i);   // the owner stored it before it entered the all-reduce: normally there
                unsigned long long spins = 0;
                while (zi.w != epoch && alive) {
                    __nanosleep(20);
                    if (++spins > q.spin_limit) { atomicAdd(q.status + 7, 1u); break; }
                    zi = ld_volatile_v4(own.z + i);
                }
                if (upd[0]) pi.x = __uint_as_float(zi.x) + beta[0] * pi.x;
                if (upd[1]) pi.y = __uint_as_float(zi.y) + beta[1] * pi.y;
                if (upd[2]) pi.z = __uint_as_float(zi.z) + beta[2] * pi.z;
                own.p[i] = pi;
            }
        }
        ++loops;
        lap(4);
        alive = mg_local_sync(q, s_last, ++lseq, alive);
        lap(5);
    }
    // x -= mean(x) (:277), then every rank gets the complete solution
    for (int k = 0; k < 6; ++k) acc[k] = 0.0;
    for (uint32_t i = q.r0 + tid; i < q.r1; i += nth)
        for (int c = 0; c < 3; ++c) acc[c] += (double)own.x[(size_t)c * R + i];
    alive = mg_allreduce6(q, acc, smem, s_last, parity, ++epoch, ++seq, false, alive, tot); parity ^= 1;
    float mean[3];
    for (int c = 0; c < 3; ++c) mean[c] = R ? (float)(tot[c] / (double)R) : 0.0f;
    for (uint32_t i = q.r0 + tid; i < q.r1; i += nth)
        for (int c = 0; c < 3; ++c) {
            const float v = own.x[(size_t)c * R + i] - mean[c];
            for (uint32_t k = 0; k < q.nranks; ++k) mg_carve(q.peer[k], R).x[(size_t)c * R + i] = v;
        }
    for (int k = 0; k < 6; ++k) acc[k] = 0.0;
    alive = mg_allreduce6(q, acc, smem, s_last, parity, ++epoch, ++seq, true, alive, tot);   // barrier: all x stored everywhere
    if (tid == 0) {
        for (int c = 0; c < 3; ++c) {
            q.status[c] = iters[c];
            const float err = rhsNorm2[c] != 0.0f ? sqrtf(resNorm2[c] / rhsNorm2[c]) : 0.0f;
            q.status[3 + c] = __float_as_uint(err);
        }
        q.status[6] = loops;
        q.status[8] = epoch;
        q.status[22] = n_imp;
    }
}

// ---- host side: peer block management and launch -----------------------------------------------------------------
struct MgState {
    void *block = nullptr;                 // own MgBlock (cudaMalloc)
    void *peer[MG_MAX_RANKS] = {nullptr};  // opened peers (peer[rank] = block)
    bool opened[MG_MAX_RANKS] = {false};
    uint32_t R = 0, rank = 0, nranks = 1, epoch = 0;
    DevBuf<double> blockpart;
    DevBuf<uint32_t> status;
    DevBuf<uint8_t> dest;     // halo destination mask of every row
    DevBuf<uint8_t> imp_mark; // rows of other ranks this rank reads
    DevBuf<uint32_t> imp, n_imp;
    uint32_t *pinned = nullptr;
};

void seam_mg_free(b2tex_ctx *c)
{
    MgState *m = c->seam_mg;
    if (!m) return;
    for (uint32_t k = 0; k < MG_MAX_RANKS; ++k)
        if (m->opened[k] && m->peer[k]) cudaIpcCloseMemHandle(m->peer[k]);
    if (m->block) cudaFree(m->block);
    if (m->pinned) cudaFreeHost(m->pinned);
    delete m;
    c->seam_mg = nullptr;
}

// assembly must have run (b2tex_seam_assemble); allocates the peer block for R rows and returns its IPC handle
int seam_mg_export(b2tex_ctx *c, uint32_t rank, uint32_t nranks, void *handle64)
{
    if (!c->R) { set_error("seam_mg_export: assemble the seam system first"); return B2TEX_ERR_ARG; }
    if (nranks < 1 || nranks > (uint32_t)MG_MAX_RANKS || rank >= nranks) { set_error("seam_mg_export: at most %d ranks", MG_MAX_RANKS); return B2TEX_ERR_ARG; }
    seam_mg_free(c);
    MgState *m = new MgState();
    c->seam_mg = m;
    m->R = c->R; m->rank = rank; m->nranks = nranks;
    const size_t bytes = mg_block_bytes(c->R);
    B2_CUDA(cudaMalloc(&m->block, bytes));
    B2_CUDA(cudaMemsetAsync(m->block, 0, bytes, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    m->peer[rank] = m->block;
    B2_TRY(m->blockpart.alloc(4096 * 8));   // every allocation happens here: nothing inside the solve waits for the device
    B2_TRY(m->status.alloc(32));
    B2_TRY(m->dest.alloc(c->R));
    B2_TRY(m->imp_mark.alloc(c->R));
    B2_TRY(m->imp.alloc(c->R));
    B2_TRY(m->n_imp.alloc(1));
    B2_CUDA(cudaHostAlloc((void **)&m->pinned, 32 * sizeof(uint32_t), cudaHostAllocDefault));
    cudaFuncAttributes fa;   // load the kernels now (the first launch of a lazily loaded kernel synchronises the context)
    B2_CUDA(cudaFuncGetAttributes(&fa, (const void *)k_pcg_mg));
    B2_CUDA(cudaFuncGetAttributes(&fa, (const void *)k_pcg_mg_dest));
    B2_CUDA(cudaFuncGetAttributes(&fa, (const void *)k_pcg_mg_imports));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    cudaIpcMemHandle_t h;
    memset(&h, 0, sizeof(h));
    if (nranks > 1) B2_CUDA(cudaIpcGetMemHandle(&h, m->block));   // a single rank has nobody to hand its block to
    memcpy(handle64, &h, 64);
    return B2TEX_OK;
}

int seam_mg_import(b2tex_ctx *c, uint32_t peer_rank, const void *handle64)
{
    MgState *m = c->seam_mg;
    if (!m || peer_rank >= m->nranks) { set_error("seam_mg_import: export first"); return B2TEX_ERR_ARG; }
    if (peer_rank == m->rank) return B2TEX_OK;
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    B2_CUDA(cudaIpcOpenMemHandle(&m->peer[peer_rank], h, cudaIpcMemLazyEnablePeerAccess));
    m->opened[peer_rank] = true;
    return B2TEX_OK;
}

// peers inside one process: attach the raw device pointer of the peer's block instead of an IPC handle
int seam_mg_attach(b2tex_ctx *c, uint32_t peer_rank, void *peer_block)
{
    MgState *m = c->seam_mg;
    if (!m || peer_rank >= m->nranks || !peer_block) { set_error("seam_mg_attach: export first"); return B2TEX_ERR_ARG; }
    if (peer_rank != m->rank) m->peer[peer_rank] = peer_block;
    return B2TEX_OK;
}
void *seam_mg_block(b2tex_ctx *c) { return c->seam_mg ? c->seam_mg->block : nullptr; }

int seam_mg_solve(b2tex_ctx *c, b2tex_seam_info *info)
{
    invalidate(c, SEAM);
    B2_TRY(require(c, SEAM_SYSTEM, "seam_mg_solve"));
    MgState *m = c->seam_mg;
    if (!m || m->R != c->R) { set_error("seam_mg_solve: export / import the peer blocks for this system first"); return B2TEX_ERR_ARG; }
    for (uint32_t k = 0; k < m->nranks; ++k)
        if (!m->peer[k]) { set_error("seam_mg_solve: peer %u not imported", k); return B2TEX_ERR_ARG; }
    cudaStream_t s = c->stream;
    const uint32_t R = c->R;
    const uint32_t r0 = (uint32_t)((uint64_t)R * m->rank / m->nranks), r1 = (uint32_t)((uint64_t)R * (m->rank + 1) / m->nranks);
    int per_sm = 0;
    B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pcg_mg, MG_THREADS, 0));
    if (per_sm < 1) { set_error("k_pcg_mg cannot be resident"); return B2TEX_ERR_CUDA; }
    int grid = c->num_sms * per_sm;
    const int need = (int)((r1 - r0 + MG_THREADS - 1) / MG_THREADS);
    if (grid > need) grid = std::max(1, need);
    if (grid > 4096) grid = 4096;
    B2_TRY(m->status.zero(s));
    PcgMg q;
    q.R = R; q.r0 = r0; q.r1 = r1; q.rank = m->rank; q.nranks = m->nranks;
    q.csr_ptr = c->csr_ptr.p; q.csr_enc = c->csr_enc.p; q.diag_val = c->seam_dval.p; q.inv_diag = c->seam_diag.p; q.rhs = c->seam_rhs.p;
    q.r = c->seam_r.p; q.t = c->seam_t.p; q.blockpart = m->blockpart.p; q.status = m->status.p; q.dest = m->dest.p;
    B2_TRY(m->imp_mark.zero(s));
    B2_TRY(m->n_imp.zero(s));
    if (r1 > r0) B2_LAUNCH k_pcg_mg_dest<<<(r1 - r0 + 255) / 256, 256, 0, s>>>(R, r0, r1, m->rank, m->nranks, c->csr_ptr.p, c->csr_enc.p, m->dest.p, m->imp_mark.p);
    B2_LAUNCH k_pcg_mg_imports<<<(R + 255) / 256, 256, 0, s>>>(R, m->imp_mark.p, m->imp.p, m->n_imp.p);
    q.imp = m->imp.p; q.n_imp = m->n_imp.p;
    for (int k = 0; k < MG_MAX_RANKS; ++k) q.peer[k] = m->peer[k];
    static const bool seam_timing = getenv("B2TEX_SEAM_TIMING") != nullptr;
    q.timing = seam_timing ? 1u : 0u;
    q.max_iters = 1000u; q.tol = 0.0001f; q.epoch0 = m->epoch; q.spin_limit = 4ull * 1000 * 1000;   // x (20 ns sleep + a system-scope load): a few seconds
    void *args[] = {&q};
    cudaEvent_t e0, e1;
    B2_CUDA(cudaEventCreate(&e0)); B2_CUDA(cudaEventCreate(&e1));
    B2_CUDA(cudaEventRecord(e0, s));
    count_launch();
    B2_CUDA(cudaLaunchCooperativeKernel((void *)k_pcg_mg, dim3(grid), dim3(MG_THREADS), args, 0, s));
    B2_CUDA(cudaEventRecord(e1, s));
    uint32_t st[32];
    // read back through pinned memory: a copy to pageable memory waits for the stream inside the driver, which (ranks driven
    // from one process) would keep the peers from launching the kernel this one is waiting for
    if (!m->pinned) B2_CUDA(cudaHostAlloc((void **)&m->pinned, 32 * sizeof(uint32_t), cudaHostAllocDefault));
    B2_CUDA(cudaMemcpyAsync(m->pinned, m->status.p, sizeof(st), cudaMemcpyDeviceToHost, s));
    // the complete solution sits in the own peer block: copy it where the single-GPU path leaves it
    B2_CUDA(cudaMemcpyAsync(c->seam_x.p, mg_carve(m->block, R).x, 3 * (size_t)R * sizeof(float), cudaMemcpyDeviceToDevice, s));
    B2_CUDA(cudaStreamSynchronize(s));
    memcpy(st, m->pinned, sizeof(st));
    float ms = 0.0f;
    cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    m->epoch = st[8];
    if (seam_timing)
        fprintf(stderr, "k_pcg_mg rank %u: %u iterations, block 0 [us]: spmv %.0f allreduce_a %.0f update %.0f allreduce_b %.0f p %.0f local_barrier %.0f; imports %u\n",
                m->rank, st[6], st[16] / 1e3, st[17] / 1e3, st[18] / 1e3, st[19] / 1e3, st[20] / 1e3, st[21] / 1e3, st[22]);
    if (st[7]) { set_error("k_pcg_mg: %u cross-GPU barrier timeouts (a peer did not arrive)", st[7]); return B2TEX_ERR_CUDA; }
    for (int ch = 0; ch < 3; ++ch) { info->iterations[ch] = st[ch]; memcpy(&info->residual[ch], &st[3 + ch], 4); }
    info->cg_launch_iterations = st[6];
    info->cg_ms = ms;
    mark_valid(c, SEAM);
    return B2TEX_OK;
}

}  // namespace b2
