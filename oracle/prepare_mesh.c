/* prepare_mesh.c -- CPU restatement of tex::prepare_mesh (libs/tex/prepare_mesh.cpp:14-70) -- TEST INFRASTRUCTURE.
 *
 * Built into its own library by oracle_prepare.py with the oracle's flags (-ffp-contract=off: no FMA contraction).
 *
 * Redundant faces (prepare_mesh.cpp:14-55).  Written the reference's way, as an independent check of the sort-based
 * kernels of csrc/prepare.cu: for face i, scan the incident faces of each of its three vertices (the vertex -> face rings,
 * faces ascending; a face with a repeated vertex is listed twice there); a face j > i whose three indices all occur among
 * the indices of i makes i redundant (:22-40, only the smaller id goes).  The test reads the original faces, so the order
 * of the scan does not matter.  Kept faces keep their order (:44-48); vertices are not touched.
 *
 * Face normals [UPSTREAM-RECALL] (MVE TriangleMesh::ensure_normals, :65): u = b - a, v = c - a,
 *   n = (u1*v2 - u2*v1, u2*v0 - u0*v2, u0*v1 - u1*v0), l = sqrtf((n0*n0 + n1*n1) + n2*n2), normal = l > 0 ? n / l : 0
 * componentwise, fp32, no FMA.
 *
 * Vertex normals [UPSTREAM-RECALL] (MVE TriangleMesh::recalc_normals, angle-weighted).  Stated convention, operation for
 * operation: all sums start at (0, 0, 0); faces are visited in ascending order; a face with fnl == 0 (fnl = l above)
 * adds nothing; otherwise for each corner j (vertex p = face[j], q = face[(j+1)%3], r = face[(j+2)%3]):
 *   e1 = q - p, e2 = r - p, l1 = sqrtf((e1x*e1x + e1y*e1y) + e1z*e1z), l2 likewise, e1 = e1 / l1, e2 = e2 / l2,
 *   d = (e1x*e2x + e1y*e2y) + e1z*e2z, d clamped to [-1, 1], angle = acosf(d),
 *   sum[p]_k = sum[p]_k + (n_k / fnl) * angle.
 * Finally len = sqrtf((sx*sx + sy*sy) + sz*sz) and normal = len > 0 ? sum / len : 0 componentwise (an unreferenced
 * vertex gets 0).  acosf is the C library's; the device's may differ from it in the last ulp.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

/* keep[F] = 1 for the faces that stay; returns the number of redundant faces */
uint32_t orc_remove_redundant_faces(const uint32_t *faces, uint32_t F, uint32_t nv, uint8_t *keep)
{
    uint32_t *ptr = (uint32_t *)calloc((size_t)nv + 1, sizeof(uint32_t));
    uint32_t *idx = (uint32_t *)malloc(sizeof(uint32_t) * (3 * (size_t)F + 1));
    uint32_t *fill = (uint32_t *)malloc(sizeof(uint32_t) * ((size_t)nv + 1));
    for (size_t i = 0; i < 3 * (size_t)F; ++i) ptr[faces[i] + 1]++;
    for (uint32_t v = 0; v < nv; ++v) ptr[v + 1] += ptr[v];
    for (uint32_t v = 0; v <= nv; ++v) fill[v] = ptr[v];
    for (uint32_t f = 0; f < F; ++f)
        for (int k = 0; k < 3; ++k) idx[fill[faces[3 * (size_t)f + k]]++] = f;
    uint32_t removed = 0;
    for (uint32_t i = 0; i < F; ++i) {
        const uint32_t *fi = faces + 3 * (size_t)i;
        int redundant = 0;
        for (int j = 0; !redundant && j < 3; ++j)
            for (uint32_t k = ptr[fi[j]]; !redundant && k < ptr[fi[j] + 1]; ++k) {
                const uint32_t g = idx[k];
                if (g <= i) continue;
                int all = 1;
                for (int l = 0; l < 3 && all; ++l) {
                    const uint32_t w = faces[3 * (size_t)g + l];
                    all = w == fi[0] || w == fi[1] || w == fi[2];
                }
                redundant = all;
            }
        keep[i] = (uint8_t)!redundant;
        removed += (uint32_t)redundant;
    }
    free(ptr); free(idx); free(fill);
    return removed;
}

static float face_cross(const float *verts, const uint32_t *f, float n[3])
{
    const float *a = verts + 3 * (size_t)f[0], *b = verts + 3 * (size_t)f[1], *c = verts + 3 * (size_t)f[2];
    const float u0 = b[0] - a[0], u1 = b[1] - a[1], u2 = b[2] - a[2];
    const float v0 = c[0] - a[0], v1 = c[1] - a[1], v2 = c[2] - a[2];
    n[0] = u1 * v2 - u2 * v1;
    n[1] = u2 * v0 - u0 * v2;
    n[2] = u0 * v1 - u1 * v0;
    return sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
}

/* out[F][3]; returns the number of zero normals */
uint32_t orc_face_normals(const float *verts, const uint32_t *faces, uint32_t F, float *out)
{
    uint32_t zero = 0;
    for (uint32_t f = 0; f < F; ++f) {
        float n[3];
        const float l = face_cross(verts, faces + 3 * (size_t)f, n);
        for (int k = 0; k < 3; ++k) out[3 * (size_t)f + k] = l > 0.0f ? n[k] / l : 0.0f;
        zero += !(l > 0.0f);
    }
    return zero;
}

/* out[nv][3] */
void orc_vertex_normals(const float *verts, uint32_t nv, const uint32_t *faces, uint32_t F, float *out)
{
    for (size_t i = 0; i < 3 * (size_t)nv; ++i) out[i] = 0.0f;
    for (uint32_t f = 0; f < F; ++f) {
        const uint32_t *id = faces + 3 * (size_t)f;
        float n[3];
        const float fnl = face_cross(verts, id, n);
        if (fnl == 0.0f) continue;
        for (int j = 0; j < 3; ++j) {
            const float *p = verts + 3 * (size_t)id[j], *q = verts + 3 * (size_t)id[(j + 1) % 3],
                        *r = verts + 3 * (size_t)id[(j + 2) % 3];
            float e1[3] = {q[0] - p[0], q[1] - p[1], q[2] - p[2]}, e2[3] = {r[0] - p[0], r[1] - p[1], r[2] - p[2]};
            const float l1 = sqrtf(e1[0] * e1[0] + e1[1] * e1[1] + e1[2] * e1[2]);
            const float l2 = sqrtf(e2[0] * e2[0] + e2[1] * e2[1] + e2[2] * e2[2]);
            for (int k = 0; k < 3; ++k) { e1[k] = e1[k] / l1; e2[k] = e2[k] / l2; }
            float d = e1[0] * e2[0] + e1[1] * e2[1] + e1[2] * e2[2];
            d = d < -1.0f ? -1.0f : (d > 1.0f ? 1.0f : d);
            const float angle = acosf(d);
            float *s = out + 3 * (size_t)id[j];
            for (int k = 0; k < 3; ++k) s[k] = s[k] + (n[k] / fnl) * angle;
        }
    }
    for (uint32_t v = 0; v < nv; ++v) {
        float *s = out + 3 * (size_t)v;
        const float len = sqrtf(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]);
        for (int k = 0; k < 3; ++k) s[k] = len > 0.0f ? s[k] / len : 0.0f;
    }
}
