// b2_types.h -- host-side types of the tex:: veneer.
//
// The reference's boundary types come from MVE (absent) and libs/tex; this header provides the minimal equivalents the
// hot-path signatures of libs/tex/texturing.h:59-106 need, with the SAME type and member names texrecon uses
// (apps/texrecon/texrecon.cpp:78-189), so that the literal call sequence of texrecon compiles against it
// (tests/cpp/texrecon_hotpath.cpp) and a maintainer can either include this header stand-alone or replace the shim
// namespaces by the real MVE headers (INTEGRATION.md).
//
// What is different behind the same names: DataCosts, UniGraph labels and TexturePatch images are HANDLES on results that
// stay resident on the GPU between the tex:: calls (tex::DeviceSession); host copies are made when an accessor asks.
#pragma once

#include <array>
#include <cstdint>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

namespace math {
template <typename T, int N>
struct Vector {
    T v[N];
    Vector() { for (int i = 0; i < N; ++i) v[i] = T(0); }
    explicit Vector(T a) { for (int i = 0; i < N; ++i) v[i] = a; }
    Vector(T a, T b) { static_assert(N == 2, "Vec2 constructor"); v[0] = a; v[1] = b; }
    Vector(T a, T b, T c) { static_assert(N == 3, "Vec3 constructor"); v[0] = a; v[1] = b; v[2] = c; }
    T &operator[](int i) { return v[i]; }
    T const &operator[](int i) const { return v[i]; }
    T *operator*() { return v; }
    T const *operator*() const { return v; }
};
typedef Vector<float, 2> Vec2f;
typedef Vector<int, 2> Vec2i;
typedef Vector<float, 3> Vec3f;
}  // namespace math

namespace mve {
/* mve::TriangleMesh: the three lists the path reads (calculate_data_costs.cpp:136-138) */
class TriangleMesh {
public:
    typedef std::shared_ptr<TriangleMesh> Ptr;
    typedef std::shared_ptr<TriangleMesh const> ConstPtr;
    typedef std::vector<math::Vec3f> VertexList;
    typedef std::vector<unsigned int> FaceList;
    typedef std::vector<math::Vec3f> NormalList;
    static Ptr create() { return Ptr(new TriangleMesh()); }
    VertexList const &get_vertices() const { return vertices; }
    VertexList &get_vertices() { return vertices; }
    FaceList const &get_faces() const { return faces; }
    FaceList &get_faces() { return faces; }
    NormalList const &get_face_normals() const { return face_normals; }
    NormalList &get_face_normals() { return face_normals; }
    /* angle-weighted vertex normals, filled by tex::prepare_mesh (texrecon's OBJ writer reads them) */
    NormalList const &get_vertex_normals() const { return vertex_normals; }
    NormalList &get_vertex_normals() { return vertex_normals; }
    /* MVE ensure_normals(face=true): normalised cross(b-a, c-a), zero for degenerate faces */
    void ensure_face_normals();
private:
    VertexList vertices;
    FaceList faces;
    NormalList face_normals, vertex_normals;
};

/* mve::MeshInfo: per-vertex incident faces and 1-ring (global_seam_leveling.cpp:55,61,161,187) */
class MeshInfo {
public:
    struct VertexInfo {
        std::vector<std::size_t> verts;
        std::vector<std::size_t> faces;
    };
    MeshInfo() {}
    explicit MeshInfo(TriangleMesh::ConstPtr mesh) { initialize(mesh); }
    void initialize(TriangleMesh::ConstPtr mesh);
    VertexInfo const &operator[](std::size_t i) const { return infos[i]; }
    std::size_t size() const { return infos.size(); }
    /* appends (build_adjacency_graph.cpp:31-34 relies on that) */
    void get_faces_for_edge(std::size_t v1, std::size_t v2, std::vector<std::size_t> *adjacent_faces) const;
private:
    std::vector<VertexInfo> infos;
    std::vector<unsigned int> const *faces = nullptr;
};

/* mve::Image<T>: width x height x channels, interleaved.  The pixels either belong to the image or are a window into a
 * buffer a tex::DeviceSession keeps alive (the patch images of one scene are one host buffer, filled by one download). */
template <typename T>
class Image {
public:
    typedef std::shared_ptr<Image<T> > Ptr;
    typedef std::shared_ptr<Image<T> const> ConstPtr;
    static Ptr create(int width, int height, int channels) { return Ptr(new Image<T>(width, height, channels)); }
    static Ptr create_view(int width, int height, int channels, T *pixels, std::shared_ptr<void> keep_alive)
    {
        Ptr p(new Image<T>());
        p->w = width; p->h = height; p->c = channels; p->ext = pixels; p->keep = keep_alive;
        return p;
    }
    int width() const { return w; }
    int height() const { return h; }
    int channels() const { return c; }
    T *get_data_pointer() { return ext ? ext : own.data(); }
    T const *get_data_pointer() const { return ext ? ext : own.data(); }
    T &at(int x, int y, int ch) { return get_data_pointer()[((std::size_t)y * w + x) * c + ch]; }
    T const &at(int x, int y, int ch) const { return get_data_pointer()[((std::size_t)y * w + x) * c + ch]; }
    T &at(std::size_t i) { return get_data_pointer()[i]; }
    T const &at(std::size_t i) const { return get_data_pointer()[i]; }
    std::size_t get_value_amount() const { return (std::size_t)w * h * c; }
private:
    Image() {}
    Image(int width, int height, int channels) : w(width), h(height), c(channels), own((std::size_t)width * height * channels) {}
    int w = 0, h = 0, c = 0;
    std::vector<T> own;
    T *ext = nullptr;
    std::shared_ptr<void> keep;
};
typedef Image<float> FloatImage;
typedef Image<std::uint8_t> ByteImage;
}  // namespace mve

namespace tex {

class DeviceSession;  // texturing.cpp: one b2tex_ctx with the scene resident on the GPU

/* libs/tex/settings.h:58-95 */
enum DataTerm { DATA_TERM_AREA = 0, DATA_TERM_GMI = 1 };
enum SmoothnessTerm { SMOOTHNESS_TERM_POTTS = 0 };
enum OutlierRemoval { OUTLIER_REMOVAL_NONE = 0, OUTLIER_REMOVAL_GAUSS_DAMPING = 1, OUTLIER_REMOVAL_GAUSS_CLAMPING = 2 };
enum ToneMapping { TONE_MAPPING_NONE = 0, TONE_MAPPING_GAMMA = 1 };
struct Settings {
    bool verbose = false;
    DataTerm data_term = DATA_TERM_GMI;
    SmoothnessTerm smoothness_term = SMOOTHNESS_TERM_POTTS;
    OutlierRemoval outlier_removal = OUTLIER_REMOVAL_NONE;
    ToneMapping tone_mapping = TONE_MAPPING_NONE;
    bool geometric_visibility_test = true;
    bool global_seam_leveling = true;
    bool local_seam_leveling = true;
    bool hole_filling = true;
    bool keep_unseen_faces = false;
};

/* libs/tex/texture_view.h:26-34 */
struct FaceProjectionInfo {
    std::uint16_t view_id;
    float quality;
    math::Vec3f mean_color;
    bool operator<(FaceProjectionInfo const &other) const { return view_id < other.view_id; }
};

/* libs/tex/seam_leveling.h:22-45 */
struct VertexProjectionInfo {
    std::size_t texture_patch_id;
    math::Vec2f projection;
    std::vector<std::size_t> faces;
    bool operator<(VertexProjectionInfo const &other) const { return texture_patch_id < other.texture_patch_id; }
};
struct EdgeProjectionInfo {
    std::size_t texture_patch_id;
    math::Vec2f p1;
    math::Vec2f p2;
    bool operator<(EdgeProjectionInfo const &other) const { return texture_patch_id < other.texture_patch_id; }
};
struct MeshEdge {
    std::size_t v1;
    std::size_t v2;
};

/* DataCosts = SparseTable<uint32 face, uint16 view, float> (texturing.h:36, sparse_table.h:29-66): same accessors.
 * Columns (faces) are stored as ONE compressed array (the reference keeps a vector per column plus a row-wise copy the
 * path never reads); tex::calculate_data_costs fills it in bulk -- or not at all: the table then is a handle on the
 * costs that stay on the GPU for tex::view_selection, and the host copy is fetched when col() is first asked for. */
template <typename C, typename R, typename T>
class SparseTable {
public:
    typedef std::pair<R, T> Entry;
    struct Column {   // what col() returns: iterable, indexable, sized -- like the reference's std::vector<pair>
        Entry const *first;
        Entry const *last;
        Entry const *begin() const { return first; }
        Entry const *end() const { return last; }
        std::size_t size() const { return (std::size_t)(last - first); }
        bool empty() const { return first == last; }
        Entry const &operator[](std::size_t i) const { return first[i]; }
    };
    SparseTable() : ncols(0), nrows(0) {}
    SparseTable(C cols, R rows) : ncols(cols), nrows(rows), ptr((std::size_t)cols + 1, 0) {}
    C cols() const { return ncols; }
    R rows() const { return nrows; }
    Column col(C id) const
    {
        fetch();
        finish_tail();
        Entry const *b = entries.data();
        return Column{b + ptr[id], b + ptr[(std::size_t)id + 1]};
    }
    /* sparse_table.h:105-110; columns must be filled in ascending order (calculate_data_costs.cpp:291-298 does) */
    void set_value(C col, R row, T value)
    {
        fetch();
        host_modified = true;
        if (col < open_col || col >= ncols) throw std::runtime_error("SparseTable::set_value: columns must be filled in ascending order");
        while (open_col < col) { ++open_col; ptr[open_col] = entries.size(); }
        entries.push_back(Entry(row, value));
        tail_dirty = true;
    }
    std::size_t get_nnz() const { return (session && !fetched) ? device_nnz : entries.size(); }
    /* bulk fill from CSR arrays (one pass, no per-entry call) */
    void assign_csr(std::uint64_t const *col_ptr, R const *row, T const *value)
    {
        session.reset(); device_nnz = 0; fetched = false;
        ptr.assign(col_ptr, col_ptr + (std::size_t)ncols + 1);
        entries.resize(ptr[ncols]);
        for (std::size_t i = 0; i < entries.size(); ++i) entries[i] = Entry(row[i], value[i]);
        open_col = ncols ? ncols - 1 : 0;
        tail_dirty = false;
    }
    /* handle on device-resident costs: (session, number of entries); see tex::calculate_data_costs */
    void attach_device(std::shared_ptr<DeviceSession> s, std::size_t nnz, unsigned generation)
    {
        session = s; device_nnz = nnz; fetched = false; host_modified = false; device_generation = generation;
        entries.clear(); open_col = 0; tail_dirty = false;
    }
    std::shared_ptr<DeviceSession> const &device_session() const { return session; }
    /* true while the device copy is the table: attached and not edited through set_value since */
    bool device_copy_valid() const { return session && !host_modified; }
    unsigned generation() const { return device_generation; }
private:
    void fetch() const;   // texturing.cpp: downloads the device-resident table once
    void finish_tail() const
    {
        if (!tail_dirty) return;
        for (std::size_t c = (std::size_t)open_col + 1; c <= ncols; ++c) ptr[c] = entries.size();
        tail_dirty = false;
    }
    C ncols;
    R nrows;
    mutable std::vector<std::uint64_t> ptr;
    mutable std::vector<Entry> entries;
    mutable C open_col = 0;
    mutable bool tail_dirty = false;
    std::shared_ptr<DeviceSession> session;
    std::size_t device_nnz = 0;
    unsigned device_generation = 0;
    bool host_modified = false;
    mutable bool fetched = false;
    friend class DeviceSession;
};
typedef SparseTable<std::uint32_t, std::uint16_t, float> DataCosts;
template <> void SparseTable<std::uint32_t, std::uint16_t, float>::fetch() const;   // texturing.cpp

/* face adjacency graph + labels (libs/tex/uni_graph.h:20-78) */
class UniGraph {
public:
    explicit UniGraph(std::size_t nodes) : adj(nodes), labels(nodes, 0), edges(0) {}
    std::size_t num_nodes() const { return adj.size(); }
    std::size_t num_edges() const { return edges; }
    bool has_edge(std::size_t a, std::size_t b) const {
        for (std::size_t x : adj[a]) if (x == b) return true;
        return false;
    }
    void add_edge(std::size_t a, std::size_t b) {
        if (has_edge(a, b)) return;
        adj[a].push_back(b); adj[b].push_back(a); ++edges;
    }
    std::vector<std::size_t> const &get_adj_nodes(std::size_t n) const { return adj[n]; }
    void set_label(std::size_t n, std::size_t l) { labels[n] = l; }
    std::size_t get_label(std::size_t n) const { return labels[n]; }
private:
    std::vector<std::vector<std::size_t> > adj;
    std::vector<std::size_t> labels;
    std::size_t edges;
};
typedef UniGraph Graph;

/* camera + image of one view (libs/tex/texture_view.h:39-52); the image is borrowed, not loaded:
 * image IO/undistortion (generate_texture_views.cpp) is out of scope */
struct TextureView {
    std::size_t id = 0;
    float pos[3] = {0, 0, 0};
    float viewdir[3] = {0, 0, 1};
    float projection[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};  // row major
    float world_to_cam[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    int width = 0, height = 0;
    std::uint8_t const *rgb = nullptr;  // H x W x 3
    std::size_t get_id() const { return id; }
    int get_width() const { return width; }
    int get_height() const { return height; }
};
typedef std::vector<TextureView> TextureViews;

}  // namespace tex

/* global namespace, like the reference's (libs/tex/texture_patch.h has no TEX_NAMESPACE; texrecon.cpp:178 writes
 * TexturePatch::Ptr unqualified) */
/* libs/tex/texture_patch.h:28-101: label, faces, texture coordinates, float image, validity and blending masks -- the
 * interface generate_texture_atlases / texture_atlas.cpp read.  Patches made by tex::generate_texture_patches are handles:
 * their pixels live in the DeviceSession's patch buffers and are refreshed from the GPU when an accessor is called after a
 * device stage (global / local seam leveling) has changed them. */
class TexturePatch {
public:
    typedef std::shared_ptr<TexturePatch> Ptr;
    typedef std::shared_ptr<const TexturePatch> ConstPtr;
    typedef std::vector<std::size_t> Faces;
    typedef std::vector<math::Vec2f> Texcoords;

    TexturePatch(int _label, Faces const &_faces, Texcoords const &_texcoords, mve::FloatImage::Ptr _image);
    static Ptr create(int label, Faces const &faces, Texcoords const &texcoords, mve::FloatImage::Ptr image)
    {
        return std::make_shared<TexturePatch>(label, faces, texcoords, image);
    }
    /* texture_patch.cpp:41-116.  Device-backed patches: zero offsets are what tex::generate_texture_patches already applied
     * (texrecon.cpp:174-183); other offsets come from tex::global_seam_leveling.  There is no host implementation. */
    void adjust_colors(std::vector<math::Vec3f> const &adjust_values);

    Faces &get_faces() { return faces; }
    Faces const &get_faces() const { return faces; }
    Texcoords &get_texcoords() { return texcoords; }
    Texcoords const &get_texcoords() const { return texcoords; }
    mve::FloatImage::Ptr get_image() { sync(); return image; }
    mve::FloatImage::ConstPtr get_image() const { sync(); return image; }
    mve::ByteImage::ConstPtr get_validity_mask() const { sync(); return validity_mask; }
    mve::ByteImage::ConstPtr get_blending_mask() const { sync(); return blending_mask; }
    int get_label() const { return label; }
    int get_width() const { return image->width(); }
    int get_height() const { return image->height(); }
    int get_size() const { return get_width() * get_height(); }
    /* view pixel of patch pixel (0, 0) (generate_texture_patches.cpp:117-121: min - texture_patch_border) */
    int get_min_x() const { return min_x; }
    int get_min_y() const { return min_y; }
    std::shared_ptr<tex::DeviceSession> const &device_session() const { return session; }
private:
    void sync() const;   // texturing.cpp
    int label;
    Faces faces;
    Texcoords texcoords;
    mve::FloatImage::Ptr image;
    mve::ByteImage::Ptr validity_mask;
    mve::ByteImage::Ptr blending_mask;
    int min_x = 0, min_y = 0;
    std::shared_ptr<tex::DeviceSession> session;
    friend class tex::DeviceSession;
};

namespace tex {

/* libs/tex/texturing.h:31-38 */
typedef std::vector<TexturePatch::Ptr> TexturePatches;
typedef std::vector<std::vector<VertexProjectionInfo> > VertexProjectionInfos;
typedef std::vector<std::vector<FaceProjectionInfo> > FaceProjectionInfos;

}  // namespace tex
