// undistort.cu -- radial undistortion of the resident rgb views (generate_texture_views.cpp:154-162).
//
// The reference undistorts the image of every .cam view with dist[0] != 0 while it loads the scene, before any stage sees
// a pixel: MVE image_undistort_k2k4 when dist[1] != 0, image_undistort_vsfm otherwise.  Here the uploaded images are
// resampled once on the device, so that every later stage (gradient, validity mask, qualities, seam colours, patches)
// reads undistorted pixels.  Arithmetic: the CPU restatement in oracle/undistort.c, operation for operation (doubles for
// the coordinates, compiled with -fmad=false), then the u8 bilinear sample of the data-cost stage.
//
// The resampling is a gather and cannot run in place, and a second copy of all images would double their footprint
// (12.4 GB per rank at C5).  The views are resampled in batches into a bounded scratch buffer and copied back.
#include <math.h>

#include <algorithm>

#include "common.cuh"
#include "sampling.cuh"

namespace b2 {

namespace {

constexpr int UPX = 4;   // output pixels per thread: 12 bytes, three aligned 32-bit stores

struct UndistortView {
    const uint8_t *src;   // the view's rgb image
    uint8_t *dst;         // its undistorted image (scratch, 16-byte aligned)
    int32_t w, h;
    int32_t k2k4;         // 1: Bundler k2 k4 model, 0: VisualSFM
    double fl, k0, k1;    // flen * max(w, h) and the two coefficients
};

// source position (pixel centres at integers) of output pixel (x, y); false where there is none
__device__ __forceinline__ bool undistort_source(int x, int y, const UndistortView &V, float *sx, float *sy)
{
    const double cx = 0.5 * (double)V.w, cy = 0.5 * (double)V.h;
    const double ux = ((double)x + 0.5 - cx) / V.fl, uy = ((double)y + 0.5 - cy) / V.fl;
    const double r2 = ux * ux + uy * uy;
    double s;
    if (V.k2k4) {
        s = 1.0 + V.k0 * r2 + V.k1 * r2 * r2;
    } else {
        // VisualSFM: the source scale s solves q s^3 + s - 1 = 0 (Newton from 1); no positive root below q = -4/27
        const double q = V.k0 * r2;
        if (27.0 * q < -4.0) return false;
        s = 1.0;
        for (int it = 0; it < 100; ++it) {
            const double sn = s - (q * s * s * s + s - 1.0) / (3.0 * q * s * s + 1.0);
            if (sn == s) break;
            s = sn;
        }
    }
    const double px = ux * s * V.fl + cx, py = uy * s * V.fl + cy;
    if (!(px >= 0.0 && px < (double)V.w && py >= 0.0 && py < (double)V.h)) return false;   // also NaN
    *sx = (float)(px - 0.5);
    *sy = (float)(py - 0.5);
    return true;
}

// blockIdx.y = view of the batch, UPX consecutive output pixels (row major) per thread.  Blocks past the end of a smaller
// view exit.  No warp collective: the serial host emulation runs it thread after thread.
__global__ void __launch_bounds__(256) k_undistort(const UndistortView *__restrict__ views)
{
    const UndistortView V = views[blockIdx.y];
    const size_t n = (size_t)V.w * V.h;
    const size_t p0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * UPX;
    if (p0 >= n) return;
    uint8_t o[3 * UPX];
#pragma unroll
    for (int j = 0; j < UPX; ++j) {
        const size_t p = p0 + j;
        const int y = (int)(p / (size_t)V.w), x = (int)(p - (size_t)y * V.w);
        float sx = 0.0f, sy = 0.0f;
        const bool in = p < n && undistort_source(x, y, V, &sx, &sy);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) o[3 * j + ch] = in ? linear_at_rgb(V.src, V.w, V.h, sx, sy, ch) : (uint8_t)0;
    }
    uint8_t *dst = V.dst + 3 * p0;   // 12 bytes per thread from a 16-byte aligned base: 4-byte aligned
    if (p0 + UPX <= n) {
        uint32_t *d = reinterpret_cast<uint32_t *>(dst);
#pragma unroll
        for (int i = 0; i < 3; ++i)
            d[i] = (uint32_t)o[4 * i] | ((uint32_t)o[4 * i + 1] << 8) | ((uint32_t)o[4 * i + 2] << 16) | ((uint32_t)o[4 * i + 3] << 24);
    } else {
        for (size_t i = 0; i < 3 * (n - p0); ++i) dst[i] = o[i];
    }
}

}  // namespace

// Scratch for one batch of resampled views.  A view larger than this gets a batch (and a scratch buffer) of its own.
constexpr size_t UNDISTORT_SCRATCH_BYTES = size_t(256) << 20;

int undistort_views(b2tex_ctx *c, const b2tex_distortion *d, uint32_t num_views)
{
    if (!c->K) { set_error("undistort_views: no views set"); return B2TEX_ERR_ARG; }
    B2_TRY(require(c, PIXELS, "undistort_views"));
    if (num_views != c->K) { set_error("undistort_views: %u distortions for %u views", num_views, c->K); return B2TEX_ERR_ARG; }
    if (!d) { set_error("undistort_views: null distortion array"); return B2TEX_ERR_ARG; }
    std::vector<uint32_t> todo;
    for (uint32_t v = 0; v < c->K; ++v) {
        if (d[v].dist[0] == 0.0f) continue;   // generate_texture_views.cpp:154: the image is used as it is
        if (!(std::isfinite(d[v].flen) && d[v].flen > 0.0f) || !std::isfinite(d[v].dist[0]) || !std::isfinite(d[v].dist[1])) {
            set_error("undistort_views: view %u: focal length %g, distortion %g %g", v, (double)d[v].flen, (double)d[v].dist[0],
                      (double)d[v].dist[1]);
            return B2TEX_ERR_ARG;
        }
        todo.push_back(v);
    }
    if (todo.empty()) return B2TEX_OK;
    invalidate(c, PIXELS);
    B2_TRY(wait_for_images(c));
    cudaStream_t s = c->stream;

    // batches of consecutive views to be resampled that fit the scratch (16-byte aligned slots)
    auto slot = [&](uint32_t v) { return (3 * (c->img_off[v + 1] - c->img_off[v]) + 15) & ~(size_t)15; };
    size_t scratch_bytes = UNDISTORT_SCRATCH_BYTES;
    for (uint32_t v : todo) scratch_bytes = std::max(scratch_bytes, slot(v));
    std::vector<UndistortView> hv(todo.size());
    std::vector<size_t> batch_begin{0};
    size_t used = 0, peak = 0;
    for (size_t i = 0; i < todo.size(); ++i) {
        const uint32_t v = todo[i];
        if (used + slot(v) > scratch_bytes) { batch_begin.push_back(i); used = 0; }
        UndistortView &u = hv[i];
        const b2tex_view &cv = c->views_host[v];
        u.src = c->rgb.p + 3 * c->img_off[v];
        u.dst = reinterpret_cast<uint8_t *>(used);   // offset into the scratch until it exists
        u.w = cv.width; u.h = cv.height;
        u.k2k4 = d[v].dist[1] != 0.0f;
        u.fl = (double)d[v].flen * (double)std::max(cv.width, cv.height);
        u.k0 = (double)d[v].dist[0]; u.k1 = (double)d[v].dist[1];
        used += slot(v);
        peak = std::max(peak, used);
    }
    batch_begin.push_back(todo.size());
    DevBuf<uint8_t> scratch;
    DevBuf<UndistortView> dv;
    B2_TRY(scratch.alloc(peak));
    for (UndistortView &u : hv) u.dst = scratch.p + reinterpret_cast<size_t>(u.dst);
    B2_TRY(dv.upload(hv.data(), hv.size(), s));
    for (size_t b = 0; b + 1 < batch_begin.size(); ++b) {
        const size_t i0 = batch_begin[b], i1 = batch_begin[b + 1];
        size_t maxpx = 0, px = 0;
        for (size_t i = i0; i < i1; ++i) {
            maxpx = std::max(maxpx, (size_t)hv[i].w * hv[i].h);
            px += (size_t)hv[i].w * hv[i].h;
        }
        {
            // 3 B gathered + 3 B written per output pixel
            ScopedTimer tm(c, "k_undistort", 6.0 * (double)px);
            dim3 grid((unsigned)((maxpx + 256 * UPX - 1) / (256 * UPX)), (unsigned)(i1 - i0));
            B2_LAUNCH k_undistort<<<grid, 256, 0, s>>>(dv.p + i0);
            B2_KERNEL_CHECK();
        }
        ScopedTimer tm(c, "undistort_copy_back", 6.0 * (double)px);
        for (size_t i = i0; i < i1; ++i)
            B2_CUDA(cudaMemcpyAsync(const_cast<uint8_t *>(hv[i].src), hv[i].dst, 3 * (size_t)hv[i].w * hv[i].h,
                                    cudaMemcpyDeviceToDevice, s));
    }
    // zero fill can blacken corners (and resampling can brighten a black one): the validity masks follow the new pixels
    std::vector<uint32_t> flags;
    B2_TRY(prepare_views(c, 0));
    B2_TRY(zero_corner_flags(c, flags));   // synchronises the stream: scratch and dv may go
    c->any_corner_flag = std::any_of(flags.begin(), flags.end(), [](uint32_t f) { return f != 0; });
    mark_valid(c, PIXELS);
    return B2TEX_OK;
}

}  // namespace b2
