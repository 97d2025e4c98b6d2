"""-m gpu: tex::prepare_mesh on the device (b2tex_prepare_mesh, csrc/prepare.cu) against the ring-scan oracle
(oracle/prepare_mesh.c): kept faces, their input ids and face normals bit for bit, vertex normals within 1e-6, the resident
graph of the kept faces, every stage after a prepare byte-identical to the same stage after set_mesh + build_mesh_graph
with the oracle's kept faces, repeated prepares on one context, and the error paths."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import oracle_prepare as OP
from test_prepare_mesh_cpu import MESHES, quirk_mesh, prep_meshes

pytestmark = pytest.mark.gpu

ARG = 3   # B2TEX_ERR_ARG


@pytest.fixture(scope="module")
def meshes(scene_mod, get_scene):
    m = prep_meshes(scene_mod, get_scene("tiny"))
    for name in ("C3s", "C5s"):
        s = scene_mod.config(name, with_images=False)
        m[name] = (s.verts, s.faces)
    m["wide"] = quirk_mesh(4, n=40, offset=4_200_000)   # 23-bit vertex ids: sets of 69 bits
    return m


def _prepare(b2, verts, faces, c=None):
    own = c is None
    c = c or b2.Context(0)
    info = c.prepare_mesh(verts, faces)
    out = c.prepared_mesh_download(info)
    out["graph"] = c.mesh_graph_download(info.graph)
    if own:
        c.close()
    return info, out


@pytest.mark.parametrize("name", MESHES + ("C3s", "C5s", "wide"))
def test_prepare_matches_the_oracle(b2, scene_mod, meshes, name):
    verts, faces = meshes[name]
    info, d = _prepare(b2, verts, faces)
    o = OP.prepare_mesh(verts, faces)
    assert info.num_faces_in == len(faces) and info.num_faces == len(o["kept"])
    assert info.num_redundant == o["num_redundant"] and info.num_zero_normals == o["num_zero_normals"]
    assert np.array_equal(d["faces"], o["faces"]) and np.array_equal(d["kept"], o["kept"])
    assert np.array_equal(d["face_normals"].view(np.uint32), o["face_normals"].view(np.uint32))
    assert np.array_equal(d["face_normals"].view(np.uint32), scene_mod.face_normals(verts, o["faces"]).view(np.uint32))
    assert np.abs(d["vertex_normals"] - o["vertex_normals"]).max(initial=0) <= 1e-6
    if name in ("tiny", "occ", "messy", "fins", "C3s", "C5s"):   # clean: the input comes back as it went in
        assert info.num_redundant == 0 and d["faces"].tobytes() == np.ascontiguousarray(faces, np.uint32).tobytes()
    ap, ai = scene_mod.face_adjacency(o["faces"])
    rings = scene_mod.vertex_rings(o["faces"], len(verts))
    for k, want in zip(("adj_ptr", "adj_idx", "vf_ptr", "vf_idx", "vv_ptr", "vv_idx"), (ap, ai, *rings)):
        assert np.array_equal(d["graph"][k], want), k
    assert info.graph.num_adjacency == len(ai) and info.graph.num_vertex_faces == 3 * len(o["kept"])


def test_vertex_normals_are_deterministic(b2, meshes):
    verts, faces = meshes["C5s"]
    a, b = _prepare(b2, verts, faces)[1], _prepare(b2, verts, faces)[1]
    assert a["vertex_normals"].tobytes() == b["vertex_normals"].tobytes()


def _inject(scene_mod, s, frac=0.01, seed=11):
    """s's faces with about frac redundant faces (duplicates in rotated and reversed order, degenerate subset faces)
    inserted at random positions"""
    rng = np.random.RandomState(seed)
    faces = [list(f) for f in s.faces]
    for k in rng.choice(len(s.faces), max(3, int(frac * len(s.faces))), replace=False):
        a, b, c = (int(x) for x in s.faces[k])
        extra = [[b, c, a], [c, b, a], [a, a, b], [c, c, c]][k % 4]
        faces.insert(rng.randint(len(faces) + 1), extra)
    return np.asarray(faces, np.uint32)


def _stages(b2, s, prepared_faces=None):
    """every stage on one context: after prepare_mesh(verts, prepared_faces), or after set_scene(s) + build_mesh_graph"""
    c = b2.Context(0)
    if prepared_faces is not None:
        c.prepare_mesh(s.verts, prepared_faces)
        c.set_views(b2.make_views(s.pos, s.viewdir, s.proj, s.w2c, s.width, s.height, s.images), s.num_views)
    else:
        c.set_scene(s)
        c.build_mesh_graph()
    info = c.data_costs_run()
    out = dict(dc=c.data_costs_download(info.nnz))
    c.view_selection_run()
    out["labels"] = c.labels_download()
    out["x"] = c.seam_download(c.seam_run())["x"]
    pi = c.texture_patches_run(True)
    out["patches"] = c.texture_patches_download(pi)
    c.local_seam_leveling_run()
    out["local"] = c.texture_patches_download(pi)
    c.close()
    return out


def test_stages_after_prepare_are_byte_identical(b2, orc, scene_mod, get_scene):
    s = get_scene("occ")
    raw = _inject(scene_mod, s)
    o = OP.prepare_mesh(s.verts, raw)
    assert o["num_redundant"] > 0
    ref = dataclasses.replace(s, faces=o["faces"], face_normals=scene_mod.face_normals(s.verts, o["faces"]))
    p, h = _stages(b2, s, raw), _stages(b2, ref)
    for k in ("face_ptr", "view", "cost"):
        assert p["dc"][k].tobytes() == h["dc"][k].tobytes(), k
    assert p["labels"].tobytes() == h["labels"].tobytes() and p["x"].tobytes() == h["x"].tobytes()
    for key in ("patches", "local"):
        assert len(p[key]) == len(h[key])
        for a, b in zip(p[key], h[key]):
            assert (a["label"], a["min_x"], a["min_y"], a["faces"]) == (b["label"], b["min_x"], b["min_y"], b["faces"])
            for k in ("texcoords", "image", "validity", "blending"):
                assert a[k].tobytes() == b[k].tobytes(), k
    od = orc.data_costs(ref)
    assert np.array_equal(p["dc"]["view"], od["view"])
    assert p["dc"]["cost"].view(np.uint32).tobytes() == od["cost"].view(np.uint32).tobytes()


def test_repeated_prepares_on_one_context(b2, scene_mod, get_scene, meshes):
    c = b2.Context(0)
    for name in ("C5s", "quirk0", "stress", "C3s", "tiny"):
        verts, faces = meshes[name]
        info, d = _prepare(b2, verts, faces, c)
        o = OP.prepare_mesh(verts, faces)
        assert c.F == len(o["kept"]) and np.array_equal(d["faces"], o["faces"]) and np.array_equal(d["kept"], o["kept"])
    # a prepare after the stages discards their results
    s = get_scene("tiny")
    c.prepare_mesh(s.verts, s.faces)
    c.set_views(b2.make_views(s.pos, s.viewdir, s.proj, s.w2c, s.width, s.height, s.images), s.num_views)
    c.data_costs_run()
    c.view_selection_run()
    si = c.seam_run()
    c.seam_download(si)
    c.prepare_mesh(*meshes["quirk1"])
    with pytest.raises(b2.B2TexError):
        c.seam_download(si)
    with pytest.raises(b2.B2TexError):
        c.view_selection_run()
    c.close()


def test_errors(b2, meshes):
    L = b2.lib()
    verts, faces = meshes["quirk0"]
    v, f = np.ascontiguousarray(verts, np.float32), np.ascontiguousarray(faces, np.uint32)
    c = b2.Context(0)
    info = b2.B2MeshPrepInfo()
    out = np.zeros(3 * len(f), np.uint32)
    assert L.b2tex_prepared_mesh_download(c._h, b2._p(out), None, None, None) == ARG   # nothing prepared yet
    assert L.b2tex_prepare_mesh(c._h, None, C.c_uint32(len(v)), b2._p(f), C.c_uint32(len(f)), C.byref(info)) == ARG
    assert L.b2tex_prepare_mesh(c._h, b2._p(v), C.c_uint32(len(v)), None, C.c_uint32(len(f)), C.byref(info)) == ARG
    assert L.b2tex_prepare_mesh(c._h, b2._p(v), C.c_uint32(len(v)), b2._p(f), C.c_uint32(0), C.byref(info)) == ARG
    c.prepare_mesh(v, f)                                   # a good prepare, then a bad one: nothing survives
    bad = f.copy()
    bad[200, 1] = len(v)
    bad[90, 2] = len(v) + 5
    with pytest.raises(b2.B2TexError, match="face 90 "):
        c.prepare_mesh(v, bad)
    assert L.b2tex_prepared_mesh_download(c._h, b2._p(out), None, None, None) == ARG
    assert L.b2tex_build_mesh_graph(c._h, None) == ARG   # no mesh
    assert L.b2tex_mesh_graph_download(c._h, None, None, None, None, None, None) == ARG
    info = c.prepare_mesh(v, f)                            # the context recovers; NULL info is fine
    assert L.b2tex_prepare_mesh(c._h, b2._p(v), C.c_uint32(len(v)), b2._p(f), C.c_uint32(len(f)), None) == 0
    assert L.b2tex_prepared_mesh_download(c._h, None, None, None, None) == 0
    c.set_mesh(v, f, np.zeros((len(f), 3), np.float32))   # set_mesh replaces the prepared mesh
    assert L.b2tex_prepared_mesh_download(c._h, b2._p(out), None, None, None) == ARG
    c.close()
