// refshim_prepare: the mve::TriangleMesh stand-in of ../../refshim/mve/mesh.h plus the one member the reference's
// prepare_mesh.cpp calls, ensure_normals (prepare_mesh.cpp:65).  Searched before oracle/refshim only when the reference's
// prepare_mesh.cpp is compiled (oracle_prepare.build_ref); see ../README.md.
#pragma once
#include <cmath>
#include <memory>
#include <vector>
#include "math/vector.h"

namespace mve {

class TriangleMesh {
public:
    typedef std::shared_ptr<TriangleMesh> Ptr;
    typedef std::shared_ptr<TriangleMesh const> ConstPtr;
    typedef unsigned int VertexID;
    typedef std::vector<math::Vec3f> VertexList;
    typedef std::vector<math::Vec3f> NormalList;
    typedef std::vector<math::Vec4f> ColorList;
    typedef std::vector<math::Vec2f> TexCoordList;
    typedef std::vector<VertexID> FaceList;

    static Ptr create() { return Ptr(new TriangleMesh()); }
    VertexList& get_vertices() { return vertices; }
    VertexList const& get_vertices() const { return vertices; }
    FaceList& get_faces() { return faces; }
    FaceList const& get_faces() const { return faces; }
    NormalList& get_face_normals() { return face_normals; }
    NormalList const& get_face_normals() const { return face_normals; }
    NormalList& get_vertex_normals() { return vertex_normals; }
    NormalList const& get_vertex_normals() const { return vertex_normals; }
    ColorList& get_vertex_colors() { return vertex_colors; }
    ColorList const& get_vertex_colors() const { return vertex_colors; }
    TexCoordList& get_vertex_texcoords() { return vertex_texcoords; }
    TexCoordList const& get_vertex_texcoords() const { return vertex_texcoords; }
    bool has_vertex_colors() const { return !vertices.empty() && vertex_colors.size() == vertices.size(); }

    /* MVE ensure_normals [UPSTREAM-RECALL], the restatement of oracle/prepare_mesh.c (operation order stated there):
     * recomputes the face normals when their count differs from the faces', the vertex normals when theirs differs from
     * the vertices' */
    void ensure_normals(bool face = true, bool vertex = true) {
        std::size_t const nf = faces.size() / 3;
        bool const do_face = face && face_normals.size() != nf, do_vertex = vertex && vertex_normals.size() != vertices.size();
        if (do_face) face_normals.assign(nf, math::Vec3f(0.0f, 0.0f, 0.0f));
        if (do_vertex) vertex_normals.assign(vertices.size(), math::Vec3f(0.0f, 0.0f, 0.0f));
        for (std::size_t f = 0; f < nf; ++f) {
            unsigned int const* id = &faces[3 * f];
            float const* a = &vertices[id[0]][0]; float const* b = &vertices[id[1]][0]; float const* c = &vertices[id[2]][0];
            float const u0 = b[0] - a[0], u1 = b[1] - a[1], u2 = b[2] - a[2], v0 = c[0] - a[0], v1 = c[1] - a[1], v2 = c[2] - a[2];
            float const n[3] = {u1 * v2 - u2 * v1, u2 * v0 - u0 * v2, u0 * v1 - u1 * v0};
            float const l = std::sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
            if (do_face) for (int k = 0; k < 3; ++k) face_normals[f][k] = l > 0.0f ? n[k] / l : 0.0f;
            if (!do_vertex || l == 0.0f) continue;
            for (int j = 0; j < 3; ++j) {
                float const* p = &vertices[id[j]][0]; float const* q = &vertices[id[(j + 1) % 3]][0];
                float const* r = &vertices[id[(j + 2) % 3]][0];
                float e1[3] = {q[0] - p[0], q[1] - p[1], q[2] - p[2]}, e2[3] = {r[0] - p[0], r[1] - p[1], r[2] - p[2]};
                float const l1 = std::sqrt(e1[0] * e1[0] + e1[1] * e1[1] + e1[2] * e1[2]);
                float const l2 = std::sqrt(e2[0] * e2[0] + e2[1] * e2[1] + e2[2] * e2[2]);
                for (int k = 0; k < 3; ++k) { e1[k] = e1[k] / l1; e2[k] = e2[k] / l2; }
                float d = e1[0] * e2[0] + e1[1] * e2[1] + e1[2] * e2[2];
                d = d < -1.0f ? -1.0f : (d > 1.0f ? 1.0f : d);
                float const angle = std::acos(d);
                for (int k = 0; k < 3; ++k) vertex_normals[id[j]][k] = vertex_normals[id[j]][k] + (n[k] / l) * angle;
            }
        }
        if (do_vertex)
            for (std::size_t v = 0; v < vertex_normals.size(); ++v) {
                math::Vec3f& s = vertex_normals[v];
                float const len = std::sqrt(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]);
                for (int k = 0; k < 3; ++k) s[k] = len > 0.0f ? s[k] / len : 0.0f;
            }
    }

private:
    VertexList vertices;
    FaceList faces;
    NormalList face_normals, vertex_normals;
    ColorList vertex_colors;
    TexCoordList vertex_texcoords;
};

}  // namespace mve
