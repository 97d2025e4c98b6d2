// texturing.cpp -- C++ veneer: the tex:: functions of libs/tex/texturing.h:59-106 on top of the C ABI (include/b2tex.h).
//
// One tex::DeviceSession = one b2tex_ctx with a scene (mesh + view images) resident on the GPU.  texrecon calls the
// stages back to back on the same mesh (apps/texrecon/texrecon.cpp:92-189), so the session of the last mesh is cached and
// every stage continues where the previous one left its results: DataCosts never leave the device between
// calculate_data_costs and view_selection, the images are uploaded once for data costs, patches and seam leveling, patch
// pixels come back when somebody reads them.
#include "texturing.h"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <limits>
#include <mutex>

#include "../../include/b2tex.h"

namespace mve {

void TriangleMesh::ensure_face_normals()
{
    std::size_t nf = faces.size() / 3;
    face_normals.resize(nf);
    for (std::size_t f = 0; f < nf; ++f) {
        math::Vec3f const &a = vertices[faces[3 * f]], &b = vertices[faces[3 * f + 1]], &c = vertices[faces[3 * f + 2]];
        float u[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, v[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]};
        float n[3] = {u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]};
        float l = std::sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
        for (int k = 0; k < 3; ++k) face_normals[f][k] = l > 0.0f ? n[k] / l : 0.0f;
    }
}

void MeshInfo::initialize(TriangleMesh::ConstPtr mesh)
{
    faces = &mesh->get_faces();
    infos.assign(mesh->get_vertices().size(), VertexInfo());
    std::size_t nf = faces->size() / 3;
    for (std::size_t f = 0; f < nf; ++f)
        for (int k = 0; k < 3; ++k) {
            std::size_t v = (*faces)[3 * f + k];
            infos[v].faces.push_back(f);
            for (int j = 0; j < 3; ++j) {
                std::size_t w = (*faces)[3 * f + j];
                if (w == v) continue;
                bool have = false;
                for (std::size_t x : infos[v].verts) have = have || x == w;
                if (!have) infos[v].verts.push_back(w);
            }
        }
}

void MeshInfo::get_faces_for_edge(std::size_t v1, std::size_t v2, std::vector<std::size_t> *out) const
{
    for (std::size_t f : infos[v1].faces)
        if ((*faces)[3 * f] == v2 || (*faces)[3 * f + 1] == v2 || (*faces)[3 * f + 2] == v2) out->push_back(f);
}

}  // namespace mve

namespace tex {

namespace {
void check(int rc)
{
    if (rc != B2TEX_OK) throw std::runtime_error(b2tex_last_error());
}

std::vector<b2tex_view> flatten_views(TextureViews const &tv)
{
    std::vector<b2tex_view> v(tv.size());
    for (std::size_t i = 0; i < tv.size(); ++i) {
        std::memcpy(v[i].pos, tv[i].pos, sizeof(v[i].pos));
        std::memcpy(v[i].viewdir, tv[i].viewdir, sizeof(v[i].viewdir));
        std::memcpy(v[i].proj, tv[i].projection, sizeof(v[i].proj));
        std::memcpy(v[i].w2c, tv[i].world_to_cam, sizeof(v[i].w2c));
        v[i].width = tv[i].width;
        v[i].height = tv[i].height;
        v[i].rgb = tv[i].rgb;
    }
    return v;
}

void flatten_graph(UniGraph const &g, std::vector<std::uint32_t> *ptr, std::vector<std::uint32_t> *idx)
{
    ptr->assign(g.num_nodes() + 1, 0);
    for (std::size_t i = 0; i < g.num_nodes(); ++i) (*ptr)[i + 1] = (*ptr)[i] + (std::uint32_t)g.get_adj_nodes(i).size();
    idx->resize((*ptr)[g.num_nodes()]);
    for (std::size_t i = 0; i < g.num_nodes(); ++i) {
        std::uint32_t o = (*ptr)[i];
        for (std::size_t a : g.get_adj_nodes(i)) (*idx)[o++] = (std::uint32_t)a;
    }
}
}  // namespace

// ---------------------------------------------------------------------------------------------------------------------
class DeviceSession : public std::enable_shared_from_this<DeviceSession> {
public:
    b2tex_ctx *ctx = nullptr;
    mve::TriangleMesh const *mesh_key = nullptr;
    std::size_t F = 0, Vn = 0, K = 0;
    std::uint8_t const *first_image = nullptr;
    bool have_adj = false, have_rings = false;
    unsigned cost_generation = 0;   // bumped by every calculate_data_costs on this session
    // texture patches: host mirrors of the device-resident patch arrays
    b2tex_patch_info pinfo{};
    std::vector<std::int32_t> desc;
    std::shared_ptr<std::vector<float> > images;
    std::shared_ptr<std::vector<std::uint8_t> > validity, blending;
    bool pixels_stale = false;   // the device holds newer patch pixels than the mirrors
    b2tex_seam_info seam_info{};

    ~DeviceSession() { if (ctx) b2tex_destroy(ctx); }

    /* the session of this mesh + these views: the cached one if it still matches, else a fresh upload */
    static std::shared_ptr<DeviceSession> obtain(mve::TriangleMesh::ConstPtr mesh, TextureViews const *views);
    static std::shared_ptr<DeviceSession> &cached() { static std::shared_ptr<DeviceSession> s; return s; }
    static std::mutex &mutex() { static std::mutex m; return m; }

    void set_graph(UniGraph const &graph)
    {
        std::vector<std::uint32_t> ap, ai;
        flatten_graph(graph, &ap, &ai);
        check(b2tex_set_adjacency(ctx, ap.data(), ai.data()));
        have_adj = true;
    }
    void set_rings(mve::MeshInfo const &mesh_info)
    {
        std::vector<std::uint32_t> vf_ptr(Vn + 1, 0), vv_ptr(Vn + 1, 0), vf_idx, vv_idx;
        for (std::size_t v = 0; v < Vn; ++v) {
            vf_ptr[v + 1] = vf_ptr[v] + (std::uint32_t)mesh_info[v].faces.size();
            vv_ptr[v + 1] = vv_ptr[v] + (std::uint32_t)mesh_info[v].verts.size();
            for (std::size_t f : mesh_info[v].faces) vf_idx.push_back((std::uint32_t)f);
            for (std::size_t w : mesh_info[v].verts) vv_idx.push_back((std::uint32_t)w);
        }
        check(b2tex_set_vertex_rings(ctx, vf_ptr.data(), vf_idx.data(), vv_ptr.data(), vv_idx.data()));
        have_rings = true;
    }
    void set_labels(UniGraph const &graph)
    {
        std::vector<std::uint32_t> labels(F);
        for (std::size_t f = 0; f < F; ++f) {
            if (graph.get_label(f) > K) throw std::runtime_error("Incorrect labeling");   // texrecon.cpp:141-153
            labels[f] = (std::uint32_t)graph.get_label(f);
        }
        check(b2tex_set_labels(ctx, labels.data()));
    }
    void fetch_costs(DataCosts const &dc) const
    {
        std::size_t const nnz = dc.device_nnz;
        std::vector<std::uint16_t> vw(nnz);
        std::vector<float> cs(nnz);
        dc.ptr.assign(F + 1, 0);
        check(b2tex_data_costs_download(ctx, dc.ptr.data(), vw.data(), cs.data(), nullptr));
        dc.entries.resize(nnz);
        for (std::size_t i = 0; i < nnz; ++i) dc.entries[i] = DataCosts::Entry(vw[i], cs[i]);
        dc.open_col = dc.ncols ? dc.ncols - 1 : 0;
        dc.tail_dirty = false;
    }
    void sync_pixels()
    {
        if (!pixels_stale) return;
        check(b2tex_texture_patches_download(ctx, nullptr, nullptr, nullptr, images->data(), validity->data(), blending->data()));
        pixels_stale = false;
    }
    void make_patches(mve::TriangleMesh::ConstPtr mesh, VertexProjectionInfos *vpi, TexturePatches *out);
};

std::shared_ptr<DeviceSession> DeviceSession::obtain(mve::TriangleMesh::ConstPtr mesh, TextureViews const *views)
{
    std::lock_guard<std::mutex> lk(mutex());
    std::size_t const F = mesh->get_faces().size() / 3, Vn = mesh->get_vertices().size();
    std::shared_ptr<DeviceSession> &c = cached();
    if (c && c->mesh_key == mesh.get() && c->F == F && c->Vn == Vn &&
        (!views || (c->K == views->size() && (views->empty() || c->first_image == (*views)[0].rgb))))
        return c;
    if (!views) throw std::runtime_error("tex: no device session for this mesh (call tex::generate_texture_patches first)");
    if (F > std::numeric_limits<std::uint32_t>::max()) throw std::runtime_error("Exeeded maximal number of faces");
    if (views->size() > std::numeric_limits<std::uint16_t>::max()) throw std::runtime_error("Exeeded maximal number of views");
    c.reset();   // frees the previous scene's GPU memory before the new one is allocated
    std::shared_ptr<DeviceSession> s(new DeviceSession());
    int device = 0;
    if (char const *e = std::getenv("B2TEX_DEVICE")) device = std::atoi(e);
    check(b2tex_create(device, &s->ctx));
    s->mesh_key = mesh.get(); s->F = F; s->Vn = Vn; s->K = views->size();
    s->first_image = views->empty() ? nullptr : (*views)[0].rgb;
    std::vector<math::Vec3f> zero_normals;
    mve::TriangleMesh::NormalList const *normals = &mesh->get_face_normals();
    if (normals->size() != F) { zero_normals.assign(F, math::Vec3f(0.0f)); normals = &zero_normals; }
    check(b2tex_set_mesh(s->ctx, F || Vn ? *mesh->get_vertices()[0] : nullptr, (std::uint32_t)Vn, mesh->get_faces().data(),
                         F ? *(*normals)[0] : nullptr, (std::uint32_t)F));
    std::vector<b2tex_view> flat = flatten_views(*views);
    check(b2tex_set_views(s->ctx, flat.data(), (std::uint32_t)flat.size()));
    c = s;
    return s;
}

template <>
void SparseTable<std::uint32_t, std::uint16_t, float>::fetch() const
{
    if (!session || fetched) return;
    if (session->cost_generation != device_generation)
        throw std::runtime_error("DataCosts: the device copy was replaced by a later tex::calculate_data_costs on the same scene");
    fetched = true;
    session->fetch_costs(*this);
}

void release_device_session()
{
    std::lock_guard<std::mutex> lk(DeviceSession::mutex());
    DeviceSession::cached().reset();
    b2tex_release_cached_contexts();
}

}  // namespace tex

// ---------------------------------------------------------------------------------------------------------------------
TexturePatch::TexturePatch(int _label, Faces const &_faces, Texcoords const &_texcoords, mve::FloatImage::Ptr _image)
    : label(_label), faces(_faces), texcoords(_texcoords), image(_image)
{
    /* texture_patch.cpp:19-27: all pixels valid, nothing to blend */
    validity_mask = mve::ByteImage::create(image->width(), image->height(), 1);
    blending_mask = mve::ByteImage::create(image->width(), image->height(), 1);
    std::fill(validity_mask->get_data_pointer(), validity_mask->get_data_pointer() + validity_mask->get_value_amount(), 255);
}

void TexturePatch::sync() const
{
    if (session) session->sync_pixels();
}

void TexturePatch::adjust_colors(std::vector<math::Vec3f> const &adjust_values)
{
    bool all_zero = true;
    for (math::Vec3f const &a : adjust_values) all_zero = all_zero && a[0] == 0.0f && a[1] == 0.0f && a[2] == 0.0f;
    if (session && all_zero) return;   // texrecon.cpp:174-183: what tex::generate_texture_patches left on the device
    throw std::runtime_error("TexturePatch::adjust_colors: per-patch offsets are applied on the GPU by "
                             "tex::global_seam_leveling (no CPU fallback)");
}

namespace tex {

void DeviceSession::make_patches(mve::TriangleMesh::ConstPtr mesh, VertexProjectionInfos *vpi, TexturePatches *out)
{
    std::size_t const n = pinfo.num_patches, T = pinfo.num_faces, P = pinfo.num_pixels;
    desc.assign(8 * std::max<std::size_t>(n, 1), 0);
    std::vector<std::uint32_t> pf(std::max<std::size_t>(T, 1));
    std::vector<float> tc(6 * std::max<std::size_t>(T, 1));
    images.reset(new std::vector<float>(3 * std::max<std::size_t>(P, 1)));
    validity.reset(new std::vector<std::uint8_t>(std::max<std::size_t>(P, 1)));
    blending.reset(new std::vector<std::uint8_t>(std::max<std::size_t>(P, 1)));
    check(b2tex_texture_patches_download(ctx, desc.data(), pf.data(), tc.data(), nullptr, nullptr, nullptr));
    pixels_stale = true;
    out->clear();
    out->reserve(n);
    std::size_t off = 0;
    std::shared_ptr<DeviceSession> self = shared_from_this();
    mve::TriangleMesh::FaceList const &mesh_faces = mesh->get_faces();
    vpi->assign(Vn, std::vector<VertexProjectionInfo>());
    for (std::size_t q = 0; q < n; ++q) {
        std::int32_t const *d = desc.data() + 8 * q;
        std::size_t const first = (std::size_t)d[5], cnt = (std::size_t)d[6], w = (std::size_t)d[3], h = (std::size_t)d[4];
        TexturePatch::Faces faces(pf.begin() + (long)first, pf.begin() + (long)(first + cnt));
        TexturePatch::Texcoords texcoords(3 * cnt);
        for (std::size_t i = 0; i < 3 * cnt; ++i) texcoords[i] = math::Vec2f(tc[2 * (3 * first + i)], tc[2 * (3 * first + i) + 1]);
        mve::FloatImage::Ptr img = mve::FloatImage::create_view((int)w, (int)h, 3, images->data() + 3 * off, images);
        TexturePatch::Ptr p = TexturePatch::create(d[0], faces, texcoords, img);
        p->validity_mask = mve::ByteImage::create_view((int)w, (int)h, 1, validity->data() + off, validity);
        p->blending_mask = mve::ByteImage::create_view((int)w, (int)h, 1, blending->data() + off, blending);
        p->min_x = d[1]; p->min_y = d[2];
        p->session = self;
        out->push_back(p);
        /* generate_texture_patches.cpp:517-531; one (vertex, patch) entry per patch after the merge of :40-65, the faces of
         * a patch arriving in patch order */
        for (std::size_t i = 0; i < cnt; ++i)
            for (std::size_t j = 0; j < 3; ++j) {
                std::size_t const vertex_id = mesh_faces[faces[i] * 3 + j];
                std::vector<VertexProjectionInfo> &infos = (*vpi)[vertex_id];
                if (!infos.empty() && infos.back().texture_patch_id == q) infos.back().faces.push_back(faces[i]);
                else infos.push_back(VertexProjectionInfo{q, texcoords[3 * i + j], {faces[i]}});
            }
        off += w * h;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
/* prepare_mesh.cpp:57-70 on a context of its own: no views exist yet when texrecon prepares the mesh (texrecon.cpp:79) */
void prepare_mesh(mve::MeshInfo *mesh_info, mve::TriangleMesh::Ptr mesh)
{
    mve::TriangleMesh::FaceList &faces = mesh->get_faces();
    std::size_t const F = faces.size() / 3, Vn = mesh->get_vertices().size();
    if (F > std::numeric_limits<std::uint32_t>::max() || Vn > std::numeric_limits<std::uint32_t>::max())
        throw std::runtime_error("Exeeded maximal number of faces");
    {   /* a cached session of this mesh would describe the faces before the preparation */
        std::lock_guard<std::mutex> lk(DeviceSession::mutex());
        if (DeviceSession::cached() && DeviceSession::cached()->mesh_key == mesh.get()) DeviceSession::cached().reset();
    }
    int device = 0;
    if (char const *e = std::getenv("B2TEX_DEVICE")) device = std::atoi(e);
    b2tex_ctx *ctx = nullptr;
    check(b2tex_create(device, &ctx));
    std::shared_ptr<b2tex_ctx> owner(ctx, b2tex_destroy);
    b2tex_mesh_prep_info info;
    check(b2tex_prepare_mesh(ctx, Vn ? *mesh->get_vertices()[0] : nullptr, (std::uint32_t)Vn, faces.data(), (std::uint32_t)F,
                             &info));
    mve::TriangleMesh::NormalList &vn = mesh->get_vertex_normals();
    bool const want_vertex = vn.size() != Vn;   /* ensure_normals recomputes only what is missing */
    std::vector<std::uint32_t> kept_faces(3 * (std::size_t)info.num_faces);
    mve::TriangleMesh::NormalList fn(info.num_faces);
    if (want_vertex) vn.assign(Vn, math::Vec3f(0.0f));
    check(b2tex_prepared_mesh_download(ctx, kept_faces.data(), info.num_faces ? *fn[0] : nullptr,
                                       want_vertex && Vn ? *vn[0] : nullptr, nullptr));
    if (info.num_redundant > 0) std::cout << "\tRemoved " << info.num_redundant << " redundant faces." << std::endl;
    faces.assign(kept_faces.begin(), kept_faces.end());
    mesh->get_face_normals().swap(fn);
    mesh_info->initialize(mesh);
}

/* build_adjacency_graph.cpp:16-53 */
void build_adjacency_graph(mve::TriangleMesh::ConstPtr mesh, mve::MeshInfo const &mesh_info, UniGraph *graph)
{
    mve::TriangleMesh::FaceList const &faces = mesh->get_faces();
    for (std::size_t f = 0; f < faces.size() / 3; ++f) {
        std::vector<std::size_t> nb;
        mesh_info.get_faces_for_edge(faces[3 * f], faces[3 * f + 1], &nb);
        mesh_info.get_faces_for_edge(faces[3 * f + 1], faces[3 * f + 2], &nb);
        mesh_info.get_faces_for_edge(faces[3 * f + 2], faces[3 * f], &nb);
        for (std::size_t g : nb)
            if (g != f) graph->add_edge(f, g);
    }
}

void calculate_data_costs(mve::TriangleMesh::ConstPtr mesh, TextureViews *texture_views,
                          Settings const &settings, DataCosts *data_costs)
{
    std::size_t const num_faces = mesh->get_faces().size() / 3;
    std::size_t const num_views = texture_views->size();
    if (num_faces > std::numeric_limits<std::uint32_t>::max()) throw std::runtime_error("Exeeded maximal number of faces");
    if (num_views > std::numeric_limits<std::uint16_t>::max()) throw std::runtime_error("Exeeded maximal number of views");
    std::shared_ptr<DeviceSession> s = DeviceSession::obtain(mesh, texture_views);
    b2tex_settings st = {(int)settings.data_term, (int)settings.outlier_removal, settings.geometric_visibility_test ? 1 : 0};
    b2tex_dc_info info;
    check(b2tex_data_costs_run(s->ctx, &st, &info));
    /* the costs stay where tex::view_selection needs them; col() / get_nnz() fetch the host copy on demand
     * (texrecon only reads it to write OUT_data_costs.spt, texrecon.cpp:102-106) */
    if (data_costs->cols() != num_faces || data_costs->rows() != num_views) *data_costs = DataCosts((std::uint32_t)num_faces, (std::uint16_t)num_views);
    data_costs->attach_device(s, (std::size_t)info.nnz, ++s->cost_generation);
}

void postprocess_face_infos(Settings const &settings, FaceProjectionInfos *projected_face_infos, DataCosts *data_costs)
{
    std::size_t const F = projected_face_infos->size();
    std::vector<std::uint64_t> fp(F + 1, 0), fp_out(F + 1, 0);
    for (std::size_t f = 0; f < F; ++f) fp[f + 1] = fp[f] + (*projected_face_infos)[f].size();
    std::size_t const n = fp[F];
    std::vector<std::uint16_t> vw(std::max<std::size_t>(n, 1)), vw_out(std::max<std::size_t>(n, 1));
    std::vector<float> q(std::max<std::size_t>(n, 1)), mc(3 * std::max<std::size_t>(n, 1)), cs(std::max<std::size_t>(n, 1));
    for (std::size_t f = 0; f < F; ++f) {
        std::vector<FaceProjectionInfo> &infos = (*projected_face_infos)[f];
        std::sort(infos.begin(), infos.end());   // calculate_data_costs.cpp:272
        std::size_t o = fp[f];
        for (FaceProjectionInfo const &i : infos) {
            vw[o] = i.view_id; q[o] = i.quality;
            mc[3 * o] = i.mean_color[0]; mc[3 * o + 1] = i.mean_color[1]; mc[3 * o + 2] = i.mean_color[2];
            ++o;
        }
    }
    b2tex_settings st = {(int)settings.data_term, (int)settings.outlier_removal, settings.geometric_visibility_test ? 1 : 0};
    b2tex_dc_info info;
    check(b2tex_postprocess_face_infos((std::uint32_t)F, fp.data(), vw.data(), q.data(),
                                       settings.outlier_removal != OUTLIER_REMOVAL_NONE ? mc.data() : nullptr, &st, fp_out.data(),
                                       vw_out.data(), cs.data(), &info));
    if (data_costs->cols() != F) *data_costs = DataCosts((std::uint32_t)F, data_costs->rows());
    data_costs->assign_csr(fp_out.data(), vw_out.data(), cs.data());
}

void view_selection(DataCosts const &data_costs, UniGraph *graph, Settings const &)
{
    std::uint32_t const F = data_costs.cols();
    std::vector<std::uint32_t> labels(F);
    b2tex_mrf_info info;
    std::shared_ptr<DeviceSession> s = data_costs.device_session();
    if (s && data_costs.device_copy_valid() && s->cost_generation == data_costs.generation()) {   // the costs are still on the GPU
        s->set_graph(*graph);
        check(b2tex_view_selection_run(s->ctx, nullptr, &info, nullptr));
        check(b2tex_labels_download(s->ctx, labels.data()));
    } else {                                       // costs from the host (e.g. loaded with -D, texrecon.cpp:107-117)
        std::vector<std::uint64_t> fp(F + 1, 0);
        for (std::uint32_t i = 0; i < F; ++i) fp[i + 1] = fp[i] + data_costs.col(i).size();
        std::vector<std::uint16_t> vw(fp[F]);
        std::vector<float> cs(fp[F]);
        for (std::uint32_t i = 0; i < F; ++i) {
            std::uint64_t o = fp[i];
            for (auto const &e : data_costs.col(i)) { vw[o] = e.first; cs[o] = e.second; ++o; }
        }
        std::vector<std::uint32_t> ap, ai;
        flatten_graph(*graph, &ap, &ai);
        b2tex_mrf_params p;
        b2tex_default_mrf_params(&p);
        p.num_views = data_costs.rows();
        check(b2tex_view_selection(F, ap.data(), ai.data(), fp.data(), vw.data(), cs.data(), &p, labels.data(), &info));
    }
    std::size_t const num_labels = (std::size_t)data_costs.rows() + 1;  // view_selection.cpp:121-131
    for (std::uint32_t i = 0; i < F; ++i) {
        if (num_labels <= labels[i]) throw std::runtime_error("Incorrect labeling");
        graph->set_label(i, labels[i]);
    }
}

void generate_texture_patches(UniGraph const &graph, mve::TriangleMesh::ConstPtr mesh, mve::MeshInfo const &mesh_info,
                              TextureViews *texture_views, Settings const &, VertexProjectionInfos *vertex_projection_infos,
                              TexturePatches *texture_patches)
{
    std::shared_ptr<DeviceSession> s = DeviceSession::obtain(mesh, texture_views);
    s->set_graph(graph);
    s->set_rings(mesh_info);
    s->set_labels(graph);   // always: the labeling may come from a file (-L, texrecon.cpp:137-158)
    /* crop + the zero-offset adjust_colors pass of texrecon.cpp:174-183 (validity / blending masks); global_seam_leveling
     * re-crops and applies the solved offsets */
    check(b2tex_texture_patches_run(s->ctx, 0, &s->pinfo));
    s->make_patches(mesh, vertex_projection_infos, texture_patches);
}

static std::shared_ptr<DeviceSession> session_of(TexturePatches const &patches)
{
    for (TexturePatch::Ptr const &p : patches)
        if (p && p->device_session()) return p->device_session();
    throw std::runtime_error("tex: these texture patches were not made by tex::generate_texture_patches (no device session)");
}

void global_seam_leveling(UniGraph const &, mve::TriangleMesh::ConstPtr, mve::MeshInfo const &, VertexProjectionInfos const &,
                          TexturePatches *texture_patches)
{
    if (texture_patches->empty()) return;
    std::shared_ptr<DeviceSession> s = session_of(*texture_patches);
    /* labels, rings and patches are resident since generate_texture_patches: assemble + solve (global_seam_leveling.cpp:
     * 150-291), then adjust_colors of every patch with the solved offsets (:293-323) */
    check(b2tex_seam_run(s->ctx, &s->seam_info));
    b2tex_patch_info pi;
    check(b2tex_texture_patches_run(s->ctx, 1, &pi));
    if (pi.num_patches != s->pinfo.num_patches || pi.num_pixels != s->pinfo.num_pixels)
        throw std::runtime_error("tex::global_seam_leveling: the patches changed since tex::generate_texture_patches");
    s->pixels_stale = true;
}

void local_seam_leveling(UniGraph const &, mve::TriangleMesh::ConstPtr, VertexProjectionInfos const &, TexturePatches *texture_patches)
{
    if (texture_patches->empty()) return;
    std::shared_ptr<DeviceSession> s = session_of(*texture_patches);
    b2tex_local_seam_info li;
    check(b2tex_local_seam_leveling_run(s->ctx, &li));
    s->pixels_stale = true;
}

void get_adjust_values(TexturePatches const &texture_patches, AdjustValues *adjust_values)
{
    std::shared_ptr<DeviceSession> s = session_of(texture_patches);
    std::size_t const R = s->seam_info.num_rows;
    std::vector<std::uint32_t> row_ptr(s->Vn + 1), row_label(std::max<std::size_t>(R, 1));
    std::vector<float> x(3 * std::max<std::size_t>(R, 1));
    check(b2tex_seam_download(s->ctx, row_ptr.data(), row_label.data(), x.data(), nullptr));
    adjust_values->assign(s->Vn, std::map<std::size_t, math::Vec3f>());
    for (std::size_t v = 0; v < s->Vn; ++v)
        for (std::uint32_t r = row_ptr[v]; r < row_ptr[v + 1]; ++r)
            (*adjust_values)[v][row_label[r]] = math::Vec3f(x[3 * r], x[3 * r + 1], x[3 * r + 2]);
}

}  // namespace tex
