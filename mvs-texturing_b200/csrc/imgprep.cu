// imgprep.cu -- K1: per-view image preparation on the device.
//   gradient magnitude = Sobel(luminance(rgb)) as u8       (reference: texture_view.cpp:102-107)
//   validity mask      = corner flood fill of zero pixels   (texture_view.cpp:42-94)
//   erosion            = 3x3 dilation of interior invalids   (texture_view.cpp:109-132, incl. the
//                        border quirk: image-border pixels are not invalidated)
//   valid4             = AND of the 4 bilinear taps          (texture_view.cpp:264-277)
// Integer/u8 outputs are bit-exact restatements; compiled with -fmad=false.
#include <cuda.h>

#include "common.cuh"

namespace b2 {

namespace {

// ---- gradient magnitude: the arithmetic both gradient kernels share, and the kernel for views of any size -------------
// MVE desaturate_luminance -> math::interpolate<uchar>: (u8)(r*.21f + g*.72f + b*.07f + .5f)
__device__ __forceinline__ uint8_t luminance_u8(uint32_t r, uint32_t g, uint32_t b)
{
    return (uint8_t)__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn((float)r, 0.21f), __fmul_rn((float)g, 0.72f)), __fmul_rn((float)b, 0.07f)),
                              0.5f);
}

// (u8)min(255, sqrt(sx^2 + sy^2)) of the integer Sobel sums.  ss < 2^24 is exact in fp32, and for ss < 255^2 the correctly
// rounded fp32 root of an integer cannot round up to the next integer (k - sqrt(k^2-1) > 1/(2k) >> ulp): its truncation
// is floor(sqrt(ss)), as the oracle's double root gives
__device__ __forceinline__ uint32_t sobel_u8(int sx, int sy)
{
    const int ss = sx * sx + sy * sy;
    return ss >= 255 * 255 ? 255u : (uint32_t)(int)__fsqrt_rn((float)ss);
}

// one view of a batched gradient: its image and its gradient magnitude
struct GradView {
    const uint8_t *rgb;
    uint8_t *grad;
    int32_t w, h;
};

// Gradient of views of any size, all in one launch (blockIdx.z = view; the grid covers the largest view).  One block =
// TW x TH output pixels.  The raw rgb rows of the tile and its 1-pixel halo are staged with aligned 32-bit loads
// (coalesced; byte loads move 3 B per thread and reach <10 % of HBM peak); a row starts at any byte, so each staged row
// keeps the offset of its first byte in its first word.  Only the view's own bytes [rgb, rgb + 3 w h) are read: a word
// that lies partly outside them is read byte by byte.  Luminance is computed from shared memory, and the gradient
// leaves as 32-bit words where the row is aligned.  32 rows per block pay the view-table load and the halo rows once
// for twice the pixels of 16 rows, which measured 4 % slower on 200 views at 1912x1080.
constexpr int TW = 128, TH = 32, RW = (3 * (TW + 2) + 3 + 3) / 4 + 1;
__global__ void __launch_bounds__(256) k_lum_sobel(const GradView *__restrict__ views)
{
    __shared__ uint32_t raw[TH + 2][RW];
    __shared__ uint8_t lum[TH + 2][TW + 4];
    __shared__ uint32_t shift_s[TH + 2];
    const GradView V = views[blockIdx.z];
    const int w = V.w, h = V.h;
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
    if (x0 >= w || y0 >= h) return;   // the whole block leaves
    const uintptr_t lo = (uintptr_t)V.rgb, hi = lo + 3 * (size_t)w * h;
    for (int i = threadIdx.x; i < (TH + 2) * RW; i += blockDim.x) {
        const int ly = i / RW, wi = i - ly * RW;
        const int gy = y0 + ly - 1;
        if (gy < 0 || gy >= h) continue;   // rows outside the view are never read
        const uintptr_t a = lo + (size_t)gy * w * 3 + (intptr_t)(3 * (x0 - 1));
        const uintptr_t al = a & ~(uintptr_t)3, wp = al + 4 * (uintptr_t)wi;
        if (wi == 0) shift_s[ly] = (uint32_t)(a - al);
        uint32_t v = 0;
        if (wp >= lo && wp + 4 <= hi)
            v = __ldg((const uint32_t *)wp);
        else
            for (int j = 0; j < 4; ++j)
                if (wp + j >= lo && wp + j < hi) v |= (uint32_t)__ldg((const uint8_t *)(wp + j)) << (8 * j);
        raw[ly][wi] = v;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < (TH + 2) * (TW + 2); i += blockDim.x) {
        const int ly = i / (TW + 2), lx = i - ly * (TW + 2);
        const int gx = x0 + lx - 1, gy = y0 + ly - 1;
        uint8_t v = 0;   // luminance 0 outside the image
        if (gx >= 0 && gx < w && gy >= 0 && gy < h) {
            const uint8_t *p = reinterpret_cast<const uint8_t *>(raw[ly]) + shift_s[ly] + 3 * lx;
            v = luminance_u8(p[0], p[1], p[2]);
        }
        lum[ly][lx] = v;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < TW * TH / 4; i += blockDim.x) {
        const int ly = i / (TW / 4), lx0 = (i - ly * (TW / 4)) * 4;
        const int gy = y0 + ly;
        if (gy >= h) continue;
        uint8_t o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int lx = lx0 + j, gx = x0 + lx;
            o[j] = 0;
            if (gx < w && !(gy == 0 || gy == h - 1 || gx == 0 || gx == w - 1)) {
                const int a = lum[ly][lx], b = lum[ly][lx + 1], c = lum[ly][lx + 2];
                const int d = lum[ly + 1][lx], f = lum[ly + 1][lx + 2];
                const int g = lum[ly + 2][lx], hh = lum[ly + 2][lx + 1], k = lum[ly + 2][lx + 2];
                o[j] = (uint8_t)sobel_u8((c - a) + 2 * (f - d) + (k - g), (g - a) + 2 * (hh - b) + (k - c));
            }
        }
        uint8_t *dst = V.grad + (size_t)gy * w + x0 + lx0;
        if (x0 + lx0 + 3 < w && (((uintptr_t)dst) & 3) == 0) {
            *reinterpret_cast<uint32_t *>(dst) = (uint32_t)o[0] | ((uint32_t)o[1] << 8) | ((uint32_t)o[2] << 16) | ((uint32_t)o[3] << 24);
        } else {
            for (int j = 0; j < 4; ++j)
                if (x0 + lx0 + j < w) dst[j] = o[j];
        }
    }
}

// ---- TMA variant: the rgb tile (+ 1 pixel halo) of a view is staged by ONE bulk tensor copy ------------------------------
// The view set is described to the TMA unit as a 3-D tensor of 32-bit words [K][H][3 W / 4] (needs W % 16 == 0: global
// strides are multiples of 16 bytes); a CTA asks for the box {104 words, TH3 + 2 rows, 1 view} that holds the
// (TW3 + 2) x (TH3 + 2) pixels it needs and waits on an mbarrier for the 14.1 KB to land; no thread issues a global
// load.  Two rules keep every box to what the TMA unit accepts: the first
// coordinate of the box starts on a 16-byte boundary of the row, so
// the box starts three words early (104 words instead of 100); and the box of an edge tile is shifted back inside the
// image instead of relying on out-of-bounds fill, the out-of-image pixels get luminance 0 explicitly, as k_lum_sobel
// gives them.  Luminance is then computed four pixels per thread from 16-byte windows of
// the raw tile, the Sobel sums four outputs per thread from six 32-bit words of the luminance tile with shared column
// and row sums, and the gradient leaves as one 32-bit word per thread.  Same integer / fp32 arithmetic, bit-exact.
constexpr int TW3 = 128, TH3 = 32;
constexpr int BOXW3 = 104;                 // words per tile row: bytes [384 bx - 16, 384 bx + 400) before the shift (16-byte aligned start)
constexpr int LUMW3 = 136;                 // luminance tile row pitch (132 pixels used)
__device__ __forceinline__ uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// The 128-byte descriptor lives in global memory.
__global__ void __launch_bounds__(256) k_lum_sobel_tma(const CUtensorMap *__restrict__ tmap, uint8_t *__restrict__ grad_all,
                                                       int w, int h, size_t view_stride_px, uint32_t *timeouts)
{
    __shared__ __align__(128) uint32_t raw[(TH3 + 2) * BOXW3];
    __shared__ __align__(16) uint8_t lum[(TH3 + 2) * LUMW3];
    __shared__ __align__(8) unsigned long long mbar;
    const int x0 = blockIdx.x * TW3, y0 = blockIdx.y * TH3;
    // wanted box start (words, rows) and the start actually used: shifted so that the box lies inside the tensor
    // (s0 stays a multiple of 4 words: 3 W / 4 and BOXW3 are)
    const int c0 = (3 * x0) / 4 - 4, c1 = y0 - 1;
    const int s0 = min(max(c0, 0), 3 * w / 4 - BOXW3), s1 = min(max(c1, 0), h - (TH3 + 2));
    const int dx = c0 - s0 + 3, dy = c1 - s1;   // word (of the byte-offset-1 layout used below) / row of the wanted box inside the staged one
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(&mbar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the initialised barrier as the async proxy (TMA) sees it
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t bytes = (TH3 + 2) * BOXW3 * 4;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(&mbar)), "r"(bytes) : "memory");
        const int c2 = (int)blockIdx.z;
        asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                     ::"r"(smem_addr(raw)), "l"(tmap), "r"(s0), "r"(s1), "r"(c2), "r"(smem_addr(&mbar)) : "memory");
    }
    {   // every thread waits for the tile (phase 0 of the barrier)
        uint32_t done = 0;
        for (uint32_t spins = 0; !done; ++spins) {
            asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                         : "=r"(done) : "r"(smem_addr(&mbar)) : "memory");
            if (spins > (1u << 22)) break;   // a copy that never lands must not hang the device
        }
        if (!done) {   // reported by the host as an error; nothing is written
            if (threadIdx.x == 0) atomicAdd(timeouts, 1u);
            return;
        }
    }
    // luminance, four pixels per thread: pixel q of group j sits at bytes 1 + 3 (4 j + q) .. of the wanted row
    for (int i = threadIdx.x; i < (TH3 + 2) * 33; i += blockDim.x) {
        const int ly = i / 33, j = i - ly * 33;
        const int gy = y0 - 1 + ly, r = ly + dy;   // image row, row in the staged box
        uint32_t out = 0;
        if (gy >= 0 && gy < h) {
            const uint32_t *rw = raw + r * BOXW3;
            const int wi = 3 * j + dx;             // words wi .. wi + 3 of the staged row; clamped where no image pixel lives
            const uint32_t w0 = rw[min(max(wi, 0), BOXW3 - 1)], w1 = rw[min(max(wi + 1, 0), BOXW3 - 1)],
                           w2 = rw[min(max(wi + 2, 0), BOXW3 - 1)], w3 = rw[min(max(wi + 3, 0), BOXW3 - 1)];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int gx = x0 - 1 + 4 * j + q;
                if (gx < 0 || gx >= w) continue;   // luminance 0 outside the image
                const int b = 1 + 3 * q;           // byte offset in the 16-byte window
                auto byte_at = [&](int o) -> uint32_t {
                    const uint32_t word = o < 4 ? w0 : (o < 8 ? w1 : (o < 12 ? w2 : w3));
                    return (word >> (8 * (o & 3))) & 0xFFu;
                };
                out |= (uint32_t)luminance_u8(byte_at(b), byte_at(b + 1), byte_at(b + 2)) << (8 * q);
            }
        }
        *reinterpret_cast<uint32_t *>(lum + ly * LUMW3 + 4 * j) = out;
    }
    __syncthreads();
    // Sobel, four outputs per thread.  lum column c = image column x0 - 1 + c.
    uint8_t *grad = grad_all + view_stride_px * blockIdx.z;
    for (int i = threadIdx.x; i < TH3 * (TW3 / 4); i += blockDim.x) {
        const int ly = i / (TW3 / 4), lx0 = (i - ly * (TW3 / 4)) * 4;
        const int gy = y0 + ly, gx0 = x0 + lx0;
        if (gy >= h || gx0 >= w) continue;
        uint32_t t[3][2];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const uint32_t *lp = reinterpret_cast<const uint32_t *>(lum + (ly + r) * LUMW3 + lx0);
            t[r][0] = lp[0]; t[r][1] = lp[1];
        }
        auto px = [&](int r, int cidx) -> int { return (int)((t[r][cidx >> 2] >> (8 * (cidx & 3))) & 0xFFu); };
        int col[6], rowt[4], rowb[4];   // column sums a + 2 d + g, row sums of the top / bottom row
#pragma unroll
        for (int cidx = 0; cidx < 6; ++cidx) col[cidx] = px(0, cidx) + 2 * px(1, cidx) + px(2, cidx);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            rowt[q] = px(0, q) + 2 * px(0, q + 1) + px(0, q + 2);
            rowb[q] = px(2, q) + 2 * px(2, q + 1) + px(2, q + 2);
        }
        uint32_t o = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int gx = gx0 + q;
            uint32_t out = 0;
            if (gx < w && !(gy == 0 || gy == h - 1 || gx == 0 || gx == w - 1))
                out = sobel_u8(col[q + 2] - col[q],    // (c - a) + 2 (f - d) + (k - g)
                               rowb[q] - rowt[q]);     // (g - a) + 2 (hh - b) + (k - c)
            o |= out << (8 * q);
        }
        uint8_t *dst = grad + (size_t)gy * w + gx0;
        if (gx0 + 3 < w) *reinterpret_cast<uint32_t *>(dst) = o;   // w % 16 == 0 and gx0 % 4 == 0: aligned
        else for (int q = 0; q < 4 && gx0 + q < w; ++q) dst[q] = (uint8_t)(o >> (8 * q));
    }
}

// the tensor map of the rgb images of a uniform view set, or false if the layout does not qualify
bool make_rgb_tensor_map(const uint8_t *rgb, int w, int h, uint32_t K, CUtensorMap *out)
{
    // the box of an edge tile is shifted back inside the image: the image must be at least one box wide and high
    if (w % 16 != 0 || (((uintptr_t)rgb) & 15u) != 0 || 3 * w / 4 < BOXW3 || h < TH3 + 2) return false;
    typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                 const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeFn encode = nullptr;
    static bool looked_up = false;
    if (!looked_up) {
        looked_up = true;
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) == cudaSuccess && qr == cudaDriverEntryPointSuccess)
            encode = (EncodeFn)fn;
    }
    if (!encode) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)(3 * (size_t)w / 4), (cuuint64_t)h, (cuuint64_t)K};
    const cuuint64_t strides[2] = {(cuuint64_t)(3 * (size_t)w), (cuuint64_t)(3 * (size_t)w * h)};   // bytes, dims 1 and 2
    const cuuint32_t box[3] = {(cuuint32_t)BOXW3, (cuuint32_t)(TH3 + 2), 1u};
    const cuuint32_t estr[3] = {1u, 1u, 1u};
    return encode(out, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, (void *)rgb, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

__global__ void k_corner_check(const ViewDev *views, int K, uint32_t *flags)
{
    int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= K) return;
    const ViewDev &V = views[v];
    int cx[4] = {0, 0, V.w - 1, V.w - 1}, cy[4] = {0, V.h - 1, 0, V.h - 1};
    uint32_t any = 0;
    for (int i = 0; i < 4; ++i) {
        const uint8_t *p = V.rgb + 3 * ((size_t)cx[i] + (size_t)cy[i] * V.w);
        if ((int)p[0] + p[1] + p[2] == 0) any = 1;
    }
    flags[v] = any;
}

// one view of a batched flood: its image and its invalid map (1 = invalid)
struct FloodView {
    const uint8_t *rgb;
    uint8_t *inv;
    int32_t w, h;
};

// thread per (view, corner)
__global__ void k_flood_seed(const FloodView *__restrict__ views, uint32_t n)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 4 * n) return;
    const FloodView V = views[i >> 2];
    const int w = V.w, h = V.h;
    int cx = (i & 2) ? w - 1 : 0, cy = (i & 1) ? h - 1 : 0;
    const uint8_t *p = V.rgb + 3 * ((size_t)cx + (size_t)cy * w);
    if ((int)p[0] + p[1] + p[2] == 0) V.inv[(size_t)cx + (size_t)cy * w] = 1;
}

// tile-local flood iteration over a batch of views (blockIdx.z = view): invalid spreads through 4-connected zero-sum
// pixels; any block that marked a pixel sets *changed
__global__ void __launch_bounds__(256) k_flood(const FloodView *__restrict__ views, uint32_t *changed)
{
    __shared__ uint8_t z[34][36], s[34][36];
    const FloodView V = views[blockIdx.z];
    const uint8_t *__restrict__ rgb = V.rgb;
    uint8_t *inv = V.inv;
    const int w = V.w, h = V.h;
    const int x0 = blockIdx.x * 32, y0 = blockIdx.y * 32;
    if (x0 >= w || y0 >= h) return;   // the grid covers the largest view of the batch; the whole block leaves
    for (int i = threadIdx.x; i < 34 * 34; i += blockDim.x) {
        int ly = i / 34, lx = i - ly * 34;
        int gx = x0 + lx - 1, gy = y0 + ly - 1;
        uint8_t zz = 0, ss = 0;
        if (gx >= 0 && gx < w && gy >= 0 && gy < h) {
            const uint8_t *p = rgb + 3 * ((size_t)gx + (size_t)gy * w);
            zz = ((int)p[0] + p[1] + p[2] == 0);
            ss = inv[(size_t)gx + (size_t)gy * w];
        }
        z[ly][lx] = zz;
        s[ly][lx] = ss;
    }
    __syncthreads();
    bool any_new = false;
    for (;;) {
        int ch = 0;
        for (int i = threadIdx.x; i < 32 * 32; i += blockDim.x) {
            int ly = i / 32 + 1, lx = (i & 31) + 1;
            if (z[ly][lx] && !s[ly][lx] && (s[ly - 1][lx] | s[ly + 1][lx] | s[ly][lx - 1] | s[ly][lx + 1])) {
                s[ly][lx] = 1;
                ch = 1;
            }
        }
        if (!__syncthreads_or(ch)) break;
        any_new = true;
    }
    if (any_new) {
        for (int i = threadIdx.x; i < 32 * 32; i += blockDim.x) {
            int ly = i / 32 + 1, lx = (i & 31) + 1;
            int gx = x0 + lx - 1, gy = y0 + ly - 1;
            if (gx < w && gy < h && s[ly][lx]) inv[(size_t)gx + (size_t)gy * w] = 1;
        }
        if (threadIdx.x == 0) *changed = 1;
    }
}

// erosion (optional) + 4-tap AND.  inv: 1 = invalid after flood fill.
__global__ void k_erode(const uint8_t *__restrict__ inv, uint8_t *__restrict__ er, int w, int h)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    uint8_t bad = inv[(size_t)x + (size_t)y * w];
    for (int j = -1; j <= 1 && !bad; ++j)
        for (int i = -1; i <= 1; ++i) {
            int nx = x + i, ny = y + j;
            // only INTERIOR invalid pixels dilate (texture_view.cpp:115-127)
            if (nx < 1 || nx > w - 2 || ny < 1 || ny > h - 2) continue;
            if (inv[(size_t)nx + (size_t)ny * w]) { bad = 1; break; }
        }
    er[(size_t)x + (size_t)y * w] = bad;
}

__global__ void k_valid4(const uint8_t *__restrict__ inv, uint8_t *__restrict__ v4, int w, int h)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    int x1 = min(x + 1, w - 1), y1 = min(y + 1, h - 1);
    uint8_t bad = inv[(size_t)x + (size_t)y * w] | inv[(size_t)x1 + (size_t)y * w]
        | inv[(size_t)x + (size_t)y1 * w] | inv[(size_t)x1 + (size_t)y1 * w];
    v4[(size_t)x + (size_t)y * w] = bad ? 0 : 1;
}

}  // namespace

// the compute stream waits for a deferred image upload (b2tex_set_views on the copy stream)
int wait_for_images(b2tex_ctx *c)
{
    if (c->images_in_flight) {
        B2_CUDA(cudaStreamWaitEvent(c->stream, c->images_uploaded, 0));
        c->images_in_flight = false;
    }
    return B2TEX_OK;
}

int zero_corner_flags(b2tex_ctx *c, std::vector<uint32_t> &flags)
{
    cudaStream_t s = c->stream;
    const uint32_t K = c->K;
    B2_TRY(c->scalars.alloc(std::max<size_t>(K + 64, 256)));
    B2_LAUNCH k_corner_check<<<(K + 127) / 128, 128, 0, s>>>(c->views_dev.p, (int)K, c->scalars.p + 64);
    B2_KERNEL_CHECK();
    flags.assign(K, 0);
    B2_CUDA(cudaMemcpyAsync(flags.data(), c->scalars.p + 64, K * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    B2_CUDA(cudaStreamSynchronize(s));
    return B2TEX_OK;
}

// Corner flood of the views fv (zeroed invalid maps): rounds of k_flood over all of them, each round one launch with one
// change counter and one host poll, until no block marks a pixel.  fv.size() <= K <= 65535 (b2tex_set_views), the limit
// of gridDim.z.
static int flood_fill(b2tex_ctx *c, const std::vector<FloodView> &fv, const FloodView *fv_dev)
{
    cudaStream_t s = c->stream;
    const uint32_t n = (uint32_t)fv.size();
    int maxw = 0, maxh = 0;
    for (const FloodView &f : fv) { maxw = std::max(maxw, (int)f.w); maxh = std::max(maxh, (int)f.h); }
    ScopedTimer tm(c, "k_flood", 0.0);
    B2_LAUNCH k_flood_seed<<<(4 * n + 127) / 128, 128, 0, s>>>(fv_dev, n);
    const dim3 fgrid((maxw + 31) / 32, (maxh + 31) / 32, n);
    for (int it = 0; it < 100000; ++it) {
        B2_CUDA(cudaMemsetAsync(c->scalars.p, 0, sizeof(uint32_t), s));
        B2_LAUNCH k_flood<<<fgrid, 256, 0, s>>>(fv_dev, c->scalars.p);
        uint32_t changed = 0;
        B2_CUDA(cudaMemcpyAsync(&changed, c->scalars.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        B2_CUDA(cudaStreamSynchronize(s));
        if (!changed) break;
    }
    B2_KERNEL_CHECK();
    return B2TEX_OK;
}

static void fill_view_block(b2tex_ctx *c, int data_term, std::vector<ViewDev> &vd)
{
    const uint32_t K = c->K;
    vd.resize(K);
    for (uint32_t v = 0; v < K; ++v) {
        const b2tex_view &hv = c->views_host[v];
        ViewDev &d = vd[v];
        for (int i = 0; i < 3; ++i) { d.pos[i] = hv.pos[i]; d.dir[i] = hv.viewdir[i]; }
        for (int i = 0; i < 9; ++i) d.proj[i] = hv.proj[i];
        for (int i = 0; i < 12; ++i) d.w2c[i] = hv.w2c[i];
        d.w = hv.width; d.h = hv.height;
        d.rgb = c->rgb.p + 3 * c->img_off[v];
        d.grad = data_term == 1 ? c->grad.p + c->img_off[v] : nullptr;
        d.valid4 = nullptr;
    }
}

// camera block of every view on the device (positions, matrices, image pointers): everything culling and the visibility
// rays need; touches no pixel
int prepare_views(b2tex_ctx *c, int data_term)
{
    if (!c->K) { set_error("prepare_images: no views set"); return B2TEX_ERR_ARG; }
    if (data_term == 1) B2_TRY(c->grad.alloc(c->img_off[c->K]));
    std::vector<ViewDev> vd;
    fill_view_block(c, data_term, vd);
    B2_TRY(c->views_dev.upload(vd.data(), c->K, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));   // vd is a local
    return B2TEX_OK;
}

int prepare_images(b2tex_ctx *c, int data_term, bool force)
{
    if (!force && (c->valid & IMAGES) && c->prepared_data_term == data_term) return B2TEX_OK;
    if (!c->K) { set_error("prepare_images: no views set"); return B2TEX_ERR_ARG; }
    invalidate(c, IMAGES);
    B2_TRY(wait_for_images(c));
    cudaStream_t s = c->stream;
    const uint32_t K = c->K;
    size_t total_px = c->img_off[K];

    if (data_term == 1) {
        B2_TRY(c->grad.alloc(total_px));
        DevBuf<GradView> gv_dev;   // k_lum_sobel's view table; freed after the timer has stopped
        ScopedTimer tm(c, "k_lum_sobel", 4.0 * (double)total_px);  // 3 B rgb read + 1 B gradient written
        const int w = c->views_host[0].width, h = c->views_host[0].height;
        bool uniform = true;
        for (uint32_t v = 1; v < K; ++v) uniform = uniform && c->views_host[v].width == w && c->views_host[v].height == h;
        alignas(64) CUtensorMap tmap;
        if (uniform && make_rgb_tensor_map(c->rgb.p, w, h, K, &tmap)) {
            // image tiles staged by the TMA unit (one bulk tensor copy per CTA), all views in one launch.  The 128-byte
            // descriptor lives in global memory (64-byte aligned), next to a counter of copies that never arrived.
            B2_TRY(c->tmap_dev.alloc(256));
            B2_CUDA(cudaMemcpyAsync(c->tmap_dev.p, &tmap, sizeof(tmap), cudaMemcpyHostToDevice, s));
            B2_CUDA(cudaMemsetAsync(c->tmap_dev.p + 128, 0, 4, s));
            B2_CUDA(cudaStreamSynchronize(s));   // tmap is a local
            dim3 grid((w + TW3 - 1) / TW3, (h + TH3 - 1) / TH3, K);
            B2_LAUNCH k_lum_sobel_tma<<<grid, 256, 0, s>>>(reinterpret_cast<const CUtensorMap *>(c->tmap_dev.p), c->grad.p, w, h, (size_t)w * h,
                                                 reinterpret_cast<uint32_t *>(c->tmap_dev.p + 128));
            {
                cudaError_t le = cudaGetLastError();
                if (le != cudaSuccess) { set_error("k_lum_sobel_tma launch: %s", cudaGetErrorString(le)); return B2TEX_ERR_CUDA; }
            }
            uint32_t timeouts = 0;
            B2_CUDA(cudaMemcpyAsync(&timeouts, c->tmap_dev.p + 128, 4, cudaMemcpyDeviceToHost, s));
            B2_CUDA(cudaStreamSynchronize(s));
            if (timeouts) { set_error("k_lum_sobel_tma: %u tile copies never arrived", timeouts); return B2TEX_ERR_CUDA; }
        } else {   // the views the TMA kernel declines, of any sizes: one launch, the grid sized for the largest view
            std::vector<GradView> gv(K);
            int maxw = 0, maxh = 0;
            for (uint32_t v = 0; v < K; ++v) {
                gv[v] = {c->rgb.p + 3 * c->img_off[v], c->grad.p + c->img_off[v], c->views_host[v].width, c->views_host[v].height};
                maxw = std::max(maxw, gv[v].w); maxh = std::max(maxh, gv[v].h);
            }
            B2_TRY(gv_dev.upload(gv.data(), K, s));
            const dim3 grid((maxw + TW - 1) / TW, (maxh + TH - 1) / TH, K);   // K <= 65535 (b2tex_set_views)
            B2_LAUNCH k_lum_sobel<<<grid, 256, 0, s>>>(gv_dev.p);
        }
        B2_KERNEL_CHECK();
    }

    // validity: only views with a zero-sum corner can have invalid pixels at all
    std::vector<ViewDev> vd;
    fill_view_block(c, data_term, vd);
    B2_TRY(c->views_dev.upload(vd.data(), K, s));
    std::vector<uint32_t> flags;
    B2_TRY(zero_corner_flags(c, flags));
    std::vector<FloodView> fv;
    size_t maxpx = 0;
    for (uint32_t v = 0; v < K; ++v) {
        if (!flags[v]) continue;
        // the flood runs in the view's slot of valid4, which k_valid4 overwrites at the end
        fv.push_back({c->rgb.p + 3 * c->img_off[v], nullptr, c->views_host[v].width, c->views_host[v].height});
        maxpx = std::max(maxpx, (size_t)c->views_host[v].width * c->views_host[v].height);
    }
    if (!fv.empty()) {
        B2_TRY(c->valid4.alloc(total_px));
        for (uint32_t v = 0, i = 0; v < K; ++v)
            if (flags[v]) fv[i++].inv = c->valid4.p + c->img_off[v];
        for (const FloodView &f : fv) B2_CUDA(cudaMemsetAsync(f.inv, 0, (size_t)f.w * f.h, s));
        DevBuf<FloodView> fv_dev;
        B2_TRY(fv_dev.upload(fv.data(), fv.size(), s));
        B2_TRY(flood_fill(c, fv, fv_dev.p));
        DevBuf<uint8_t> er;
        B2_TRY(er.alloc(maxpx));
        for (uint32_t v = 0; v < K; ++v) {
            if (!flags[v]) continue;
            int w = c->views_host[v].width, h = c->views_host[v].height;
            uint8_t *inv = c->valid4.p + c->img_off[v];
            dim3 b(32, 8), g((w + 31) / 32, (h + 7) / 8);
            if (data_term == 1) B2_LAUNCH k_erode<<<g, b, 0, s>>>(inv, er.p, w, h);
            else B2_CUDA(cudaMemcpyAsync(er.p, inv, (size_t)w * h, cudaMemcpyDeviceToDevice, s));
            B2_LAUNCH k_valid4<<<g, b, 0, s>>>(er.p, inv, w, h);
            B2_KERNEL_CHECK();
            vd[v].valid4 = inv;
        }
        B2_CUDA(cudaStreamSynchronize(s));
        B2_TRY(c->views_dev.upload(vd.data(), K, s));
        B2_CUDA(cudaStreamSynchronize(s));  // vd is a local
    } else {
        B2_CUDA(cudaStreamSynchronize(s));
    }
    c->prepared_data_term = data_term;
    mark_valid(c, IMAGES);
    return B2TEX_OK;
}

}  // namespace b2
