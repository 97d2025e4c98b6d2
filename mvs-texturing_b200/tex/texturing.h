// texturing.h -- the tex:: hot-path API of libs/tex/texturing.h:59-106 with the reference's signatures, backed by
// libb2tex.so (include/b2tex.h):
//
//   prepare_mesh              texturing.h:46       b2tex_prepare_mesh            (redundant faces, face + vertex normals)
//   build_adjacency_graph     texturing.h:59-61    host (feeds view_selection)
//   calculate_data_costs      texturing.h:66-69    b2tex_data_costs_run          (costs stay on the GPU)
//   postprocess_face_infos    texturing.h:71-74    b2tex_postprocess_face_infos
//   view_selection            texturing.h:79-80    b2tex_view_selection_run / b2tex_view_selection
//   generate_texture_patches  texturing.h:85-91    b2tex_texture_patches_run     (seen faces; no hole filling)
//   global_seam_leveling      texturing.h:97-101   b2tex_seam_run + b2tex_texture_patches_run(apply_adjust)
//   local_seam_leveling       texturing.h:103-106  b2tex_local_seam_leveling_run
//
// tests/cpp/texrecon_hotpath.cpp is the call sequence of apps/texrecon/texrecon.cpp:92-189 written against this header.
// The scene (mesh, images) is uploaded once per mesh: the calls share one tex::DeviceSession, DataCosts / labels /
// TexturePatches are handles on device-resident results, host copies are made when an accessor asks for them.
// Errors: std::runtime_error with the reference's messages (calculate_data_costs.cpp:315-318, view_selection.cpp:126-128);
// CUDA failures also surface as std::runtime_error.  There is no CPU fallback.
#pragma once
#include "b2_types.h"

namespace tex {

/* texrecon.cpp:79: drops the redundant faces, sets the face normals of the kept faces and (when the mesh holds none) the
 * vertex normals, re-initialises mesh_info and prints "\tRemoved N redundant faces." when N > 0 */
void
prepare_mesh(mve::MeshInfo * mesh_info, mve::TriangleMesh::Ptr mesh);

void build_adjacency_graph(mve::TriangleMesh::ConstPtr mesh, mve::MeshInfo const &mesh_info, UniGraph *graph);

void calculate_data_costs(mve::TriangleMesh::ConstPtr mesh, TextureViews *texture_views,
                          Settings const &settings, DataCosts *data_costs);

void postprocess_face_infos(Settings const &settings, FaceProjectionInfos *projected_face_infos,
                            DataCosts *data_costs);

void view_selection(DataCosts const &data_costs, UniGraph *graph, Settings const &settings);

void generate_texture_patches(UniGraph const &graph, mve::TriangleMesh::ConstPtr mesh,
                              mve::MeshInfo const &mesh_info, TextureViews *texture_views,
                              Settings const &settings, VertexProjectionInfos *vertex_projection_infos,
                              TexturePatches *texture_patches);

void global_seam_leveling(UniGraph const &graph, mve::TriangleMesh::ConstPtr mesh,
                          mve::MeshInfo const &mesh_info, VertexProjectionInfos const &vertex_projection_infos,
                          TexturePatches *texture_patches);

void local_seam_leveling(UniGraph const &graph, mve::TriangleMesh::ConstPtr mesh,
                         VertexProjectionInfos const &vertex_projection_infos, TexturePatches *texture_patches);

/* ---- additions (not in the reference) ---- */
/* per-(vertex,label) colour adjustment of the last tex::global_seam_leveling (global_seam_leveling.cpp:251,283-289) */
typedef std::vector<std::map<std::size_t, math::Vec3f> > AdjustValues;
void get_adjust_values(TexturePatches const &texture_patches, AdjustValues *adjust_values);
/* frees the cached device session (GPU memory of the last scene) */
void release_device_session();

}  // namespace tex
