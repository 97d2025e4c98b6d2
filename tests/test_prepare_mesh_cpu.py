"""tex::prepare_mesh restated on the CPU (oracle/prepare_mesh.c): the redundancy rule of prepare_mesh.cpp:14-55 against
what the reference's own translation unit returns (tests/golden/prepare_mesh_ref.npz), hand-counted 5-face meshes, face
normals bit for bit against scene.face_normals and properties of the angle-weighted vertex normals.

quirk_mesh is the seeded generator the device tests (test_emul_prepare.py, test_gpu_prepare.py) share: triple duplicates
in rotated, reversed and the same order, degenerate subset faces before and after their triangle, a pair-set face removed
by a later singleton, and a last face that copies an earlier one (the last face always survives)."""
import os

import numpy as np
import pytest

import graph_meshes as GM
import oracle_prepare as OP
import refpin

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "prepare_mesh_ref.npz")


def quirk_mesh(seed=0, n=12, offset=0):
    """(verts f32[Vn, 3], faces u32[F, 3]) on a jittered n x n grid; offset unreferenced vertices come first."""
    rng = np.random.RandomState(seed)
    g = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 2).astype(np.float64)
    verts = np.concatenate([g + rng.uniform(-0.2, 0.2, g.shape), rng.uniform(-0.3, 0.3, (len(g), 1))], 1)
    faces = []
    for i in range(n - 1):
        for j in range(n - 1):
            a, b, c, d = i * n + j, i * n + j + 1, (i + 1) * n + j, (i + 1) * n + j + 1
            faces += [[a, b, d], [a, d, c]]
    faces = [faces[k] for k in rng.permutation(len(faces))]
    tris = [list(faces[k]) for k in rng.choice(len(faces), 17, replace=False)]

    def insert(face, lo=0, hi=None):
        pos = rng.randint(lo, (len(faces) if hi is None else hi) + 1)
        faces.insert(pos, list(face))
        return pos

    for a, b, c in tris[0:6]:      # triple duplicates: rotated, reversed, same order
        for f in ([b, c, a], [c, b, a], [a, b, c]):
            insert(f)
    for a, b, c in tris[6:10]:     # a degenerate subset face before its triangle: both stay
        insert([a, a, b], 0, faces.index([a, b, c]))
    for k, (a, b, c) in enumerate(tris[10:14]):   # ... and after it: the triangle goes
        insert([[b, a, a], [a, b, a], [c, c, c], [a, c, c]][k], faces.index([a, b, c]) + 1)
    for a, b, _ in tris[14:17]:    # a pair-set face removed by a later singleton
        insert([b, b, b], insert([a, b, b]) + 1)
    faces.append(list(faces[rng.randint(len(faces))]))   # the last face copies an earlier one
    faces = np.asarray(faces, np.int64) + offset
    verts = np.concatenate([np.zeros((offset, 3)), verts], 0)
    return np.ascontiguousarray(verts, np.float32), np.ascontiguousarray(faces, np.uint32)


def prep_meshes(scene_mod, tiny):
    """name -> (verts, faces) of every mesh the golden file records"""
    out = {}
    for name in ("tiny", "occ", "messy"):
        s = scene_mod.config(name, with_images=False)
        out[name] = (s.verts, s.faces)
    for name, (faces, nv) in (("fins", GM.fin_mesh(tiny)), ("stress", GM.stress_mesh(tiny))):
        v = np.concatenate([tiny.verts, np.random.RandomState(3).uniform(-1, 1, (nv - len(tiny.verts), 3))], 0)
        out[name] = (np.ascontiguousarray(v, np.float32), faces)
    for seed in (0, 1, 2):
        out[f"quirk{seed}"] = quirk_mesh(seed)
    return out


MESHES = ("tiny", "occ", "messy", "fins", "stress", "quirk0", "quirk1", "quirk2")


@pytest.fixture(scope="module")
def meshes(scene_mod, get_scene):
    return prep_meshes(scene_mod, get_scene("tiny"))


@pytest.mark.parametrize("name", MESHES)
def test_redundant_faces_match_reference_tu(meshes, name):
    verts, faces = meshes[name]
    kf, kept, n = OP.remove_redundant_faces(faces, len(verts))
    g = np.load(GOLDEN)
    assert n == int(g[f"{name}/num_redundant"])
    assert refpin.digest(kf) == str(g[f"{name}/faces"])
    assert np.array_equal(kf, faces[kept])
    if name in ("tiny", "occ", "messy", "fins"):   # fins share edges, but no face repeats another's vertices
        assert n == 0 and np.array_equal(kf, faces)
    else:
        assert n > 0


def test_quirk_mesh_covers_every_case(meshes):
    verts, faces = meshes["quirk0"]
    _, kept, n = OP.remove_redundant_faces(faces, len(verts))
    assert kept[-1] == len(faces) - 1
    s = np.sort(faces.astype(np.int64), 1)
    assert ((s[:, 0] == s[:, 1]) & (s[:, 1] == s[:, 2])).any()
    key = s[:, 0] * 10 ** 8 + s[:, 1] * 10 ** 4 + s[:, 2]
    assert np.bincount(np.unique(key, return_inverse=True)[1]).max() >= 4   # a triangle four times
    assert n >= 6 * 3 + 4 + 3 + 1


@pytest.mark.parametrize("faces,removed,kept", [
    ([[0, 1, 2], [2, 1, 0], [1, 2, 3], [0, 1, 2], [3, 4, 5]], 2, [2, 3, 4]),        # duplicates: the highest id stays
    ([[0, 1, 2], [0, 0, 1], [1, 2, 3], [2, 3, 4], [1, 1, 1]], 3, [3, 4]),           # later degenerate subsets
    ([[0, 0, 1], [0, 1, 2], [1, 2, 3], [1, 3, 2], [3, 3, 3]], 2, [0, 1, 4]),        # an earlier subset changes nothing
    ([[0, 1, 1], [1, 1, 0], [1, 1, 1], [2, 3, 4], [4, 3, 2]], 3, [2, 4]),           # a pair set, then a singleton
    ([[0, 1, 2], [3, 4, 5], [0, 1, 3], [1, 2, 4], [5, 4, 3]], 1, [0, 2, 3, 4]),     # sharing edges is not enough
])
def test_hand_counted_five_face_meshes(faces, removed, kept):
    f = np.array(faces, np.uint32)
    kf, k, n = OP.remove_redundant_faces(f, 6)
    assert n == removed and k.tolist() == kept and np.array_equal(kf, f[kept])


@pytest.mark.parametrize("name", MESHES)
def test_face_normals_are_scene_face_normals_bit_for_bit(scene_mod, meshes, name):
    verts, faces = meshes[name]
    fn, z = OP.face_normals(verts, faces)
    want = scene_mod.face_normals(verts, faces)
    assert np.array_equal(fn.view(np.uint32), want.view(np.uint32))
    assert z == int((np.abs(want).sum(1) == 0).sum())


@pytest.mark.parametrize("name", MESHES)
def test_vertex_normals_are_unit_or_zero(meshes, name):
    verts, faces = meshes[name]
    r = OP.prepare_mesh(verts, faces)
    vn = r["vertex_normals"].astype(np.float64)
    ln = np.linalg.norm(vn, axis=1)
    assert np.all((ln == 0) | (np.abs(ln - 1) < 1e-6))
    used = np.zeros(len(verts), bool)
    used[r["faces"].ravel()] = True
    assert np.all(ln[~used] == 0)


def test_vertex_normals_of_an_octahedron_are_analytic():
    """Closed regular solid: by symmetry every vertex normal is the vertex direction."""
    v = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32)
    f = np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]], np.uint32)
    r = OP.prepare_mesh(np.concatenate([v, [[7, 7, 7]]], 0).astype(np.float32), f)
    assert r["num_redundant"] == 0
    assert np.allclose(r["vertex_normals"][:6], v, atol=1e-6) and np.all(r["vertex_normals"][6] == 0)
    assert np.allclose(r["face_normals"], np.sign(v[f].sum(1)) / np.sqrt(3), atol=1e-6)
