/* oracle/undistort.c -- TEST INFRASTRUCTURE (see oracle.h).  The image of a .cam view as texturing sees it.
 *
 * generate_texture_views.cpp:154-162 undistorts every view with dist[0] != 0 while it loads the scene, with MVE's
 * image_undistort_k2k4 (dist[1] != 0) or image_undistort_vsfm.  MVE's source is not part of the reference tree: both models
 * are restated below from its published behaviour and are UNPINNED, like the other [UPSTREAM-RECALL] pieces oracle.h lists.
 *
 * Built into its own library with bvh.c and imgprep.c (oracle_undistort.py, same flags as the Makefile).  The final sample is the oracle's own u8
 * bilinear lookup: datacosts.c is compiled into this translation unit for its linear_at_rgb, so that the data-cost stage
 * and the undistortion share one definition. */
#include "datacosts.c"

/* generate_texture_views.cpp:154-162: k0 == 0: a copy (whatever k1 is); k1 != 0: image_undistort_k2k4(flen, k0, k1);
 * otherwise image_undistort_vsfm(flen, k0).  flen is normalised by the larger image side (.cam line 2).  out must not
 * alias rgb. */
void orc_undistort(const uint8_t *rgb, int w, int h, float flen, float k0, float k1, uint8_t *out);


/* MVE image_undistort_k2k4 / image_undistort_vsfm [UPSTREAM-RECALL], chosen as generate_texture_views.cpp:154-162 does.
 * Conventions (the device kernel k_undistort repeats them operation for operation):
 *  - pixel centres: output pixel (x, y) sits at (x + 0.5, y + 0.5) in continuous image coordinates, the principal point
 *    at the image centre (w / 2, h / 2); normalised coordinates divide by fl = flen * max(w, h)
 *  - every coordinate operation is a double, evaluated left to right as written; the source position is rounded to
 *    float once, for linear_at
 *  - k2k4 (Bundler): the distorted source of the undistorted point u is u * (1 + k2 r^2 + k4 r^4), r = |u|
 *  - VisualSFM: undistorted = distorted * (1 + k r_d^2).  The source is u * s where s solves q s^3 + s - 1 = 0,
 *    q = k r^2: Newton from s = 1 until the iterate stops changing, at most 100 steps (monotone: from above for q > 0,
 *    from below for q < 0).  For q < -4/27 the cubic has no positive root: no source, the pixel stays 0
 *  - a source outside [0, w) x [0, h) leaves all three channels 0; inside, linear_at samples at (source - 0.5), i.e.
 *    clamps to the edge pixels within half a pixel of the border */
static int undistort_source(int x, int y, int w, int h, double fl, double k0, double k1, int k2k4, float *sx, float *sy)
{
    const double cx = 0.5 * (double)w, cy = 0.5 * (double)h;
    const double ux = ((double)x + 0.5 - cx) / fl, uy = ((double)y + 0.5 - cy) / fl;
    const double r2 = ux * ux + uy * uy;
    double s;
    if (k2k4) {
        s = 1.0 + k0 * r2 + k1 * r2 * r2;
    } else {
        const double q = k0 * r2;
        if (27.0 * q < -4.0) return 0;
        s = 1.0;
        for (int it = 0; it < 100; ++it) {
            const double sn = s - (q * s * s * s + s - 1.0) / (3.0 * q * s * s + 1.0);
            if (sn == s) break;
            s = sn;
        }
    }
    const double px = ux * s * fl + cx, py = uy * s * fl + cy;
    if (!(px >= 0.0 && px < (double)w && py >= 0.0 && py < (double)h)) return 0;   /* also NaN */
    *sx = (float)(px - 0.5);
    *sy = (float)(py - 0.5);
    return 1;
}

void orc_undistort(const uint8_t *rgb, int w, int h, float flen, float k0, float k1, uint8_t *out)
{
    const size_t n = (size_t)w * h;
    if (k0 == 0.0f) { memcpy(out, rgb, 3 * n); return; }
    const int k2k4 = k1 != 0.0f;
    const double fl = (double)flen * (double)(w > h ? w : h);
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            uint8_t *o = out + 3 * ((size_t)x + (size_t)y * w);
            float sx, sy;
            if (!undistort_source(x, y, w, h, fl, (double)k0, (double)k1, k2k4, &sx, &sy)) { o[0] = o[1] = o[2] = 0; continue; }
            for (int ch = 0; ch < 3; ++ch) o[ch] = linear_at_rgb(rgb, w, h, sx, sy, ch);
        }
}
