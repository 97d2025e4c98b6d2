"""tex::prepare_mesh in the C++ veneer (mvs-texturing_b200/tex): the declaration of libs/tex/texturing.h:46, a driver
that compiles with -Wall -Werror against it, and on a GPU texrecon's load-time preparation of a sphere with duplicated,
reversed and degenerate faces followed by calculate_data_costs and view_selection."""
import os
import re
import subprocess

import numpy as np
import pytest

import oracle_prepare as OP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "_prepare_mesh_veneer")


def _driver_faces(n=12):
    """the faces prepare_mesh_veneer.cpp builds: a UV sphere of n rings, a reversed copy of every 10th face, (a, a, b) after
    every 40th"""
    m = 2 * n
    ring = lambda i, j: 1 + (i - 1) * m + j % m
    south = 1 + (n - 1) * m
    F = [(0, ring(1, j), ring(1, j + 1)) for j in range(m)]
    for i in range(1, n - 1):
        for j in range(m):
            F += [(ring(i, j), ring(i + 1, j), ring(i + 1, j + 1)), (ring(i, j), ring(i + 1, j + 1), ring(i, j + 1))]
    F += [(ring(n - 1, j), south, ring(n - 1, j + 1)) for j in range(m)]
    clean = len(F)
    for f in range(0, clean, 10):
        a, b, c = F[f]
        F.append((c, b, a))
        if f % 40 == 0:
            F.append((a, a, b))
    return np.array(F, np.uint32), south + 1


def _build(b2):
    b2.lib()
    pkg = os.path.join(ROOT, "mvs-texturing_b200")
    subprocess.check_call(["/usr/bin/g++", "-std=c++11", "-O2", "-Wall", "-Werror", "-o", EXE,
                           os.path.join(ROOT, "tests", "cpp", "prepare_mesh_veneer.cpp"), os.path.join(pkg, "tex", "texturing.cpp"),
                           "-L" + pkg, "-lb2tex", "-Wl,-rpath," + pkg])


def test_declaration_matches_the_reference_header_token_for_token():
    tokens = lambda s: re.findall(r"\w+|::|[^\s\w]", s)
    want = tokens("void\nprepare_mesh(mve::MeshInfo * mesh_info, mve::TriangleMesh::Ptr mesh);")
    got = tokens(open(os.path.join(ROOT, "mvs-texturing_b200", "tex", "texturing.h")).read())
    assert any(got[i:i + len(want)] == want for i in range(len(got)))


def test_driver_compiles_and_links(b2):
    _build(b2)
    r = subprocess.run([EXE, "--link-only"], capture_output=True, text=True)
    assert r.returncode == 0 and f"input faces: {len(_driver_faces()[0])}" in r.stdout


@pytest.mark.gpu
def test_driver_prepares_and_selects_views_on_gpu(b2, scene_mod):
    _build(b2)
    r = subprocess.run([EXE], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    faces, nv = _driver_faces()
    kept, _, removed = OP.remove_redundant_faces(faces, nv)
    assert removed > 0 and f"\tRemoved {removed} redundant faces." in r.stdout
    f = {k: int(v) for k, v in re.findall(r"(\w+)=(\d+)", r.stdout)}
    assert f["removed"] == removed and f["faces"] == f["face_normals"] == len(kept)
    assert f["vertex_normals"] == f["vertices"] == nv
    # the host graph of the kept faces: every edge of scene.face_adjacency, plus the links the veneer's MeshInfo makes
    # across the repeated vertex of a kept degenerate face
    assert f["edges"] >= len(scene_mod.face_adjacency(kept)[1]) // 2
    assert f["unseen"] < len(kept)
