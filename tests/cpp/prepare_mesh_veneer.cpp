// prepare_mesh_veneer.cpp -- texrecon's load-time preparation (apps/texrecon/texrecon.cpp:78-79) followed by the first two
// stages (:97-121), written against the tex:: veneer: a sphere with duplicated, reversed and degenerate faces goes through
// tex::prepare_mesh, tex::calculate_data_costs and tex::view_selection.
//
//   prepare_mesh_veneer --link-only   no GPU needed: the calls compile and link against libb2tex.so
//   prepare_mesh_veneer               prints "removed=R faces=F face_normals=N vertex_normals=M unseen=U"
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../mvs-texturing_b200/tex/texturing.h"

namespace {

// UV sphere of radius 1: n rings of 2n segments, poles included
mve::TriangleMesh::Ptr make_sphere(int n)
{
    mve::TriangleMesh::Ptr mesh = mve::TriangleMesh::create();
    std::vector<math::Vec3f> &V = mesh->get_vertices();
    std::vector<unsigned int> &F = mesh->get_faces();
    int const m = 2 * n;
    V.push_back(math::Vec3f(0, 0, 1));
    for (int i = 1; i < n; ++i)
        for (int j = 0; j < m; ++j) {
            float const t = 3.14159265f * i / n, p = 6.2831853f * j / m;
            V.push_back(math::Vec3f(std::sin(t) * std::cos(p), std::sin(t) * std::sin(p), std::cos(t)));
        }
    V.push_back(math::Vec3f(0, 0, -1));
    unsigned const south = (unsigned)V.size() - 1;
    auto ring = [&](int i, int j) { return 1u + (unsigned)((i - 1) * m + (j % m)); };
    auto tri = [&](unsigned a, unsigned b, unsigned c) { F.push_back(a); F.push_back(b); F.push_back(c); };
    for (int j = 0; j < m; ++j) tri(0, ring(1, j), ring(1, j + 1));
    for (int i = 1; i + 1 < n; ++i)
        for (int j = 0; j < m; ++j) {
            tri(ring(i, j), ring(i + 1, j), ring(i + 1, j + 1));
            tri(ring(i, j), ring(i + 1, j + 1), ring(i, j + 1));
        }
    for (int j = 0; j < m; ++j) tri(ring(n - 1, j), south, ring(n - 1, j + 1));
    return mesh;
}

void look_at(tex::TextureView &tv, float const pos[3], float f, int W, int H)
{
    float const n = std::sqrt(pos[0] * pos[0] + pos[1] * pos[1] + pos[2] * pos[2]);
    float const zc[3] = {-pos[0] / n, -pos[1] / n, -pos[2] / n};
    float up[3] = {0, 0, 1};
    if (std::fabs(zc[2]) > 0.9f) { up[0] = 0; up[1] = 1; up[2] = 0; }
    float xc[3] = {zc[1] * up[2] - zc[2] * up[1], zc[2] * up[0] - zc[0] * up[2], zc[0] * up[1] - zc[1] * up[0]};
    float const xn = std::sqrt(xc[0] * xc[0] + xc[1] * xc[1] + xc[2] * xc[2]);
    for (float &c : xc) c /= xn;
    float const yc[3] = {zc[1] * xc[2] - zc[2] * xc[1], zc[2] * xc[0] - zc[0] * xc[2], zc[0] * xc[1] - zc[1] * xc[0]};
    float const *R[3] = {xc, yc, zc};
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) tv.world_to_cam[4 * r + c] = R[r][c];
        tv.world_to_cam[4 * r + 3] = -(R[r][0] * pos[0] + R[r][1] * pos[1] + R[r][2] * pos[2]);
    }
    for (int c = 0; c < 3; ++c) { tv.pos[c] = pos[c]; tv.viewdir[c] = zc[c]; }
    float const P[9] = {f, 0, W / 2.0f, 0, f, H / 2.0f, 0, 0, 1};
    std::memcpy(tv.projection, P, sizeof(P));
    tv.width = W; tv.height = H;
}

}  // namespace

int main(int argc, char **argv)
{
    bool const link_only = argc > 1 && !std::strcmp(argv[1], "--link-only");
    mve::TriangleMesh::Ptr mesh = make_sphere(12);
    std::vector<unsigned int> &F = mesh->get_faces();
    std::size_t const clean = F.size() / 3;
    for (std::size_t f = 0; f < clean; f += 10) {   // a reversed copy of every 10th face, a degenerate one after every 40th
        unsigned const a = F[3 * f], b = F[3 * f + 1], c = F[3 * f + 2];
        F.push_back(c); F.push_back(b); F.push_back(a);
        if (f % 40 == 0) { F.push_back(a); F.push_back(a); F.push_back(b); }
    }
    mve::MeshInfo mesh_info(mesh);                                            /* texrecon.cpp:78 */
    std::printf("input faces: %zu\n", F.size() / 3);
    if (link_only) return 0;

    try {
        std::size_t const before = F.size() / 3;
        tex::prepare_mesh(&mesh_info, mesh);                                  /* texrecon.cpp:79 */
        std::size_t const num_faces = F.size() / 3;

        int const W = 320, H = 240;
        std::size_t const num_views = 10;
        std::vector<std::vector<unsigned char> > images(num_views, std::vector<unsigned char>((std::size_t)W * H * 3));
        tex::TextureViews texture_views(num_views);
        for (std::size_t k = 0; k < num_views; ++k) {
            for (std::size_t i = 0; i < images[k].size(); ++i)
                images[k][i] = (unsigned char)(60 + (i * 7 + k * 13) % 160);
            float const t = (k + 0.5f) / num_views, phi = 2.399963f * k, z = 1.0f - 2.0f * t;
            float const r = std::sqrt(std::max(0.0f, 1.0f - z * z));
            float const pos[3] = {3 * r * std::cos(phi), 3 * r * std::sin(phi), 3 * z};
            look_at(texture_views[k], pos, 260.0f, W, H);
            texture_views[k].rgb = images[k].data();
            texture_views[k].id = k;
        }
        tex::Graph graph(num_faces);                                          /* texrecon.cpp:91-92 */
        tex::build_adjacency_graph(mesh, mesh_info, &graph);
        tex::Settings settings;
        tex::DataCosts data_costs(num_faces, texture_views.size());           /* texrecon.cpp:97-121 */
        tex::calculate_data_costs(mesh, &texture_views, settings, &data_costs);
        tex::view_selection(data_costs, &graph, settings);
        std::size_t unseen = 0;
        for (std::size_t f = 0; f < num_faces; ++f) unseen += graph.get_label(f) == 0;
        std::printf("removed=%zu faces=%zu face_normals=%zu vertex_normals=%zu vertices=%zu edges=%zu unseen=%zu\n",
                    before - num_faces, num_faces, mesh->get_face_normals().size(), mesh->get_vertex_normals().size(),
                    mesh->get_vertices().size(), graph.num_edges(), unseen);
        tex::release_device_session();
    } catch (std::exception const &e) {
        std::printf("error: %s\n", e.what());
        return 2;
    }
    return 0;
}
