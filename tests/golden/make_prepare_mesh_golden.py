"""Generates tests/golden/prepare_mesh_ref.npz: what the reference's own tex::remove_redundant_faces
(libs/tex/prepare_mesh.cpp:14-55, in oracle/_ref/libprepref.so, built by oracle_prepare.build_ref() from a checkout of
nmoehrle/mvs-texturing) returns on the meshes of tests/test_prepare_mesh_cpu.py: per mesh the digest of the kept faces
(oracle/refpin.py: digest) and the number removed.  The shim's MeshInfo gets its vertex -> face rings from
scene.vertex_rings.

    B2TEX_REFERENCE=<checkout of mvs-texturing> python tests/golden/make_prepare_mesh_golden.py
"""
import ctypes as C
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
import oracle_prepare as OP  # noqa: E402
import refpin as R  # noqa: E402
from test_prepare_mesh_cpu import GOLDEN, MESHES, prep_meshes  # noqa: E402

scene = importlib.import_module("mvs-texturing_b200.scene")
so = OP.build_ref()
if so is None:
    sys.exit("oracle/_ref/libprepref.so missing: set B2TEX_REFERENCE to a checkout of the reference")
L = C.CDLL(so)
L.ref_remove_redundant_faces.restype = C.c_uint32
out = {}
meshes = prep_meshes(scene, scene.config("tiny", with_images=False))
for name in MESHES:
    verts, faces = meshes[name]
    faces = np.ascontiguousarray(faces, np.uint32)
    rings = [np.ascontiguousarray(a, np.uint32) for a in scene.vertex_rings(faces, len(verts))[:2]]
    kept = np.zeros_like(faces)
    n = int(L.ref_remove_redundant_faces(R._p(faces), C.c_uint32(len(faces)), C.c_uint32(len(verts)), *map(R._p, rings),
                                         R._p(kept)))
    out[f"{name}/faces"] = R.digest(kept[:len(faces) - n])
    out[f"{name}/num_redundant"] = n
    print(f"{name}: {len(faces)} faces, {n} removed")
np.savez_compressed(GOLDEN, **out)
print("wrote", GOLDEN)
