/* oracle/ref_prepare_glue.cpp -- TEST INFRASTRUCTURE (see oracle.h, refshim_prepare/README.md).
 *
 * C entry point over the reference's own prepare_mesh.cpp (compiled unmodified from the reference's libs/tex against
 * oracle/refshim_prepare + oracle/refshim), so that tests can pin the oracle's redundant-face rule against the code it
 * restates.  Built by oracle_prepare.build_ref() into oracle/_ref/libprepref.so; never linked or loaded by the product path.
 */
#include <algorithm>
#include <cstdint>

#include "tex/texturing.h"

namespace tex {   /* prepare_mesh.cpp:14, not declared in texturing.h */
std::size_t remove_redundant_faces(mve::MeshInfo const& mesh_info, mve::TriangleMesh::Ptr mesh);
}

extern "C" {

/* tex::remove_redundant_faces (prepare_mesh.cpp:14-55) with the shim's MeshInfo filled from the vertex -> face rings: the
 * kept faces go to faces_out (room for 3 * num_faces entries); returns the number of faces removed */
uint32_t ref_remove_redundant_faces(const uint32_t* faces, uint32_t num_faces, uint32_t num_verts, const uint32_t* vf_ptr,
                                    const uint32_t* vf_idx, uint32_t* faces_out)
{
    mve::TriangleMesh::Ptr mesh = mve::TriangleMesh::create();
    mesh->get_faces().assign(faces, faces + 3 * static_cast<std::size_t>(num_faces));
    mve::MeshInfo mi;
    mi.resize(num_verts);
    for (uint32_t v = 0; v < num_verts; ++v) {
        mi[v].vclass = mve::MeshInfo::VERTEX_CLASS_SIMPLE;
        mi[v].faces.assign(vf_idx + vf_ptr[v], vf_idx + vf_ptr[v + 1]);
    }
    std::size_t const n = tex::remove_redundant_faces(mi, mesh);
    std::copy(mesh->get_faces().begin(), mesh->get_faces().end(), faces_out);
    return static_cast<uint32_t>(n);
}

}  // extern "C"
