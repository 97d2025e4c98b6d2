"""-m gpu: the mesh graph derived on the device (b2tex_build_mesh_graph, csrc/graph.cu) against scene.face_adjacency /
scene.vertex_rings element for element, every stage run on a derived graph against the same stage on uploaded arrays
(byte-identical outputs), the one-shot entry points with NULL topology, and the error paths."""
import ctypes as C

import numpy as np
import pytest

import graph_meshes as GM

pytestmark = pytest.mark.gpu

ARG = 3   # B2TEX_ERR_ARG


def _mesh(scene_mod, get_scene, name):
    """(verts, faces, normals) of a named scene or of the fin / stress meshes"""
    if name in ("fins", "stress"):
        faces, nv = (GM.fin_mesh if name == "fins" else GM.stress_mesh)(get_scene("tiny"))
        verts = np.random.RandomState(3).rand(nv, 3).astype(np.float32)
        return verts, faces, np.zeros((len(faces), 3), np.float32)
    s = scene_mod.config(name, with_images=False)
    return s.verts, s.faces, s.face_normals


def _check_graph(scene_mod, faces, nv, info, g):
    ap, ai = scene_mod.face_adjacency(faces)
    vf_ptr, vf_idx, vv_ptr, vv_idx = scene_mod.vertex_rings(faces, nv)
    for k, want in dict(adj_ptr=ap, adj_idx=ai, vf_ptr=vf_ptr, vf_idx=vf_idx, vv_ptr=vv_ptr, vv_idx=vv_idx).items():
        assert g[k].dtype == want.dtype and np.array_equal(g[k], want), k
    assert info.num_adjacency == len(ai) and info.num_vertex_faces == len(vf_idx)
    assert info.num_vertex_neighbours == len(vv_idx)
    assert info.max_face_degree == int(np.diff(ap.astype(np.int64)).max())
    assert info.num_non_manifold_edges == GM.non_manifold_edges(faces)


@pytest.mark.parametrize("name", ["tiny", "small", "occ", "occ2", "messy", "C2s", "C3s", "C5s", "fins", "stress"])
def test_device_graph_equals_host_arrays(b2, scene_mod, get_scene, name):
    verts, faces, normals = _mesh(scene_mod, get_scene, name)
    c = b2.Context(0)
    c.set_mesh(verts, faces, normals)
    info = c.build_mesh_graph()
    _check_graph(scene_mod, faces, verts.shape[0], info, c.mesh_graph_download(info))
    c.close()


def test_rebuild_on_one_context_with_other_sizes(b2, scene_mod, get_scene):
    """the grow-only scratch of a larger mesh serves smaller ones, and a larger one after them grows it"""
    c = b2.Context(0)
    for name in ("C3s", "tiny", "stress", "C5s", "messy"):
        verts, faces, normals = _mesh(scene_mod, get_scene, name)
        c.set_mesh(verts, faces, normals)
        info = c.build_mesh_graph()
        _check_graph(scene_mod, faces, verts.shape[0], info, c.mesh_graph_download(info))
    c.close()


def _all_stages(b2, s, graph):
    """data costs, view selection, global seam leveling, patches, local seam leveling on one context"""
    c = b2.Context(0)
    c.set_scene(s)
    if graph is None:
        c.build_mesh_graph()
    else:
        c.set_adjacency(*graph[:2])
        c.set_vertex_rings(*graph[2:])
    c.data_costs_run()
    mi, trace = c.view_selection_run()
    out = dict(labels=c.labels_download(), iterations=mi.iterations, energy=c.mrf_energy(),
               trace=trace.view(np.uint64).copy())
    si = c.seam_run()
    out["seam"] = c.seam_download(si)
    out["matrix"] = c.seam_matrix(si)
    pi = c.texture_patches_run(True)
    out["patches"] = c.texture_patches_download(pi)
    c.local_seam_leveling_run()
    out["local"] = c.texture_patches_download(pi)
    c.close()
    return out


def _same_patches(a, b):
    assert len(a) == len(b)
    for p, q in zip(a, b):
        assert (p["label"], p["min_x"], p["min_y"], p["faces"]) == (q["label"], q["min_x"], q["min_y"], q["faces"])
        for k in ("texcoords", "image", "validity", "blending"):
            assert p[k].tobytes() == q[k].tobytes(), k


@pytest.mark.parametrize("name", ["occ", "messy"])
def test_every_stage_on_the_derived_graph_is_byte_identical(b2, scene_mod, get_scene, name):
    s = get_scene(name)
    host = (*scene_mod.face_adjacency(s.faces), *scene_mod.vertex_rings(s.faces, s.verts.shape[0]))
    a, d = _all_stages(b2, s, host), _all_stages(b2, s, None)
    assert np.array_equal(a["labels"], d["labels"]) and a["iterations"] == d["iterations"]
    assert a["energy"] == d["energy"] and np.array_equal(a["trace"], d["trace"])
    for k in ("row_ptr", "row_label"):
        assert np.array_equal(a["seam"][k], d["seam"][k])
    assert a["seam"]["x"].tobytes() == d["seam"]["x"].tobytes()
    for x, y in zip(a["matrix"], d["matrix"]):
        assert x.tobytes() == y.tobytes()
    _same_patches(a["patches"], d["patches"])
    _same_patches(a["local"], d["local"])


def _patches_oneshot(b2, s, labels, topo):
    """b2tex_seam_leveling_patches (global + local leveling); topo = the six host arrays, None = six NULL pointers, or a
    list with some entries None"""
    L = b2.lib()
    views = b2.make_views(s.pos, s.viewdir, s.proj, s.w2c, s.width, s.height, s.images)
    v, f = b2._c(s.verts, np.float32), b2._c(s.faces, np.uint32)
    arrs = [None] * 6 if topo is None else [None if a is None else b2._c(a, np.uint32) for a in topo]
    lab = b2._c(labels, np.uint32)
    ptrs = [C.c_void_p() for _ in range(5)]
    pi, si, li = b2.B2PatchInfo(), b2.B2SeamInfo(), b2.B2LocalSeamInfo()
    rc = L.b2tex_seam_leveling_patches(b2._p(v), C.c_uint32(v.shape[0]), b2._p(f), C.c_uint32(f.shape[0]),
                                       *(b2._p(a) for a in arrs), b2._p(lab), views, C.c_uint32(s.num_views), C.c_int(1),
                                       C.c_int(1), *(C.byref(p) for p in ptrs), C.byref(pi), C.byref(si), C.byref(li))
    if rc:
        return rc, None
    n, T, P = int(pi.num_patches), int(pi.num_faces), int(pi.num_pixels)
    out = [b2._grab(ptrs[0], C.c_int32, 8 * n), b2._grab(ptrs[1], C.c_uint32, T), b2._grab(ptrs[2], C.c_float, 6 * T),
           b2._grab(ptrs[3], C.c_float, 3 * P), b2._grab(ptrs[4], C.c_uint8, P)]
    return 0, out


@pytest.mark.parametrize("name", ["occ", "messy"])
def test_one_shot_entry_points_with_null_topology(b2, scene_mod, get_scene, name):
    s = get_scene(name)
    adj = scene_mod.face_adjacency(s.faces)
    rings = scene_mod.vertex_rings(s.faces, s.verts.shape[0])
    h, d = b2.texture_hot_path(s, adj, rings), b2.texture_hot_path(s, None, None)
    assert np.array_equal(h["labels"], d["labels"]) and np.array_equal(h["row_ptr"], d["row_ptr"])
    assert np.array_equal(h["row_label"], d["row_label"]) and h["x"].tobytes() == d["x"].tobytes()
    assert h["mrf_info"].iterations == d["mrf_info"].iterations
    labels = h["labels"]
    gh, gd = b2.global_seam_leveling(s, rings, labels), b2.global_seam_leveling(s, None, labels)
    assert np.array_equal(gh["row_ptr"], gd["row_ptr"]) and np.array_equal(gh["row_label"], gd["row_label"])
    assert gh["x"].tobytes() == gd["x"].tobytes()
    rc_h, ph = _patches_oneshot(b2, s, labels, [*adj, *rings])
    rc_d, pd = _patches_oneshot(b2, s, labels, None)
    assert rc_h == 0 and rc_d == 0
    for x, y in zip(ph, pd):
        assert x.tobytes() == y.tobytes()


def test_errors(b2, scene_mod, get_scene):
    s = get_scene("tiny")
    nv = s.verts.shape[0]
    c = b2.Context(0)
    with pytest.raises(b2.B2TexError) as e:      # no mesh
        c.build_mesh_graph()
    assert e.value.rc == ARG
    bad = s.faces.copy()
    bad[123, 1] = nv + 2
    bad[200, 0] = nv
    c.set_mesh(s.verts, bad, s.face_normals)
    with pytest.raises(b2.B2TexError) as e:      # a face index >= Vn, the first such face named
        c.build_mesh_graph()
    assert e.value.rc == ARG and "face 123 " in str(e.value)
    with pytest.raises(b2.B2TexError) as e:      # the failed build left no graph behind
        c.mesh_graph_download(b2.B2GraphInfo())
    assert e.value.rc == ARG
    c.set_scene(s)                               # the context still works
    info = c.build_mesh_graph()
    _check_graph(scene_mod, s.faces, nv, info, c.mesh_graph_download(info))
    labels = b2.texture_hot_path(s, None, None)["labels"]
    c.set_labels(labels)
    c.seam_run()

    other = get_scene("small")                   # a new mesh drops the graph until it is rebuilt
    c.set_scene(other)
    with pytest.raises(b2.B2TexError) as e:
        c.mesh_graph_download(info)
    assert e.value.rc == ARG
    c.set_labels(np.ones(other.num_faces, np.uint32))
    with pytest.raises(b2.B2TexError) as e:
        c.seam_run()
    assert e.value.rc == ARG
    info = c.build_mesh_graph()
    c.seam_run()
    _check_graph(scene_mod, other.faces, other.verts.shape[0], info, c.mesh_graph_download(info))
    c.close()

    adj = scene_mod.face_adjacency(s.faces)
    rings = scene_mod.vertex_rings(s.faces, nv)
    with pytest.raises(b2.B2TexError) as e:      # mixed NULL topology in the one-shot calls
        b2.texture_hot_path(s, adj, None)
    assert e.value.rc == ARG
    with pytest.raises(b2.B2TexError) as e:
        b2.global_seam_leveling(s, [rings[0], None, rings[2], rings[3]], labels)
    assert e.value.rc == ARG
    rc, _ = _patches_oneshot(b2, s, labels, [*adj, None, *rings[1:]])
    assert rc == ARG
    assert b2.texture_hot_path(s, adj, rings)["labels"].tobytes() == labels.tobytes()   # the pool is still healthy
