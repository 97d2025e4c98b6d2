"""-m gpu: what a change of one resident input does to the results derived from it (csrc/state.h, include/b2tex.h).  After
the whole sequence (data costs, view selection, seam leveling, texture patches, local leveling) one input changes; every
download or stage that depends on it is refused with B2TEX_ERR_ARG, the independent ones still return what they returned
before, and re-running the stages gives byte for byte what a fresh context with the same inputs gives."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ARG = 3   # B2TEX_ERR_ARG
# per view (flen, k0, k1): pincushion distortion, so that undistorting really changes the pixels
PINCUSHION = [(0.9, 0.12, 0.03), (1.0, -0.15, 0.0), (0.8, 0.1, 0.05)]


def _views(b2, s, k=None):
    k = s.num_views if k is None else k
    return b2.make_views(s.pos[:k], s.viewdir[:k], s.proj[:k], s.w2c[:k], s.width, s.height, s.images[:k]), k


def _distortion(K):
    return (np.array([PINCUSHION[v % 3][0] for v in range(K)], np.float32),
            np.array([PINCUSHION[v % 3][1:] for v in range(K)], np.float32))


def _graph(c, scene_mod, s):
    c.set_adjacency(*scene_mod.face_adjacency(s.faces))
    c.set_vertex_rings(*scene_mod.vertex_rings(s.faces, s.verts.shape[0]))


def _stages(c):
    info = c.data_costs_run()
    out = dict(dc=c.data_costs_download(info.nnz))
    c.view_selection_run()
    out["labels"] = c.labels_download()
    sinfo = c.seam_run()
    out["seam"] = c.seam_download(sinfo)
    pinfo = c.texture_patches_run(apply_adjust=True)
    c.local_seam_leveling_run()
    out["patches"] = c.texture_patches_download(pinfo)
    return out, (info, sinfo, pinfo)


def _fresh(b2, scene_mod, s, k=None, undistort=False):
    c = b2.Context(0)
    c.set_mesh(s.verts, s.faces, s.face_normals)
    c.set_views(*_views(b2, s, k))
    if undistort:
        c.undistort_views(*_distortion(c.K))
    _graph(c, scene_mod, s)
    out, _ = _stages(c)
    c.close()
    return out


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, list):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    return a == b


# change -> (downloads and stages refused afterwards, downloads that still return what they returned before)
CASES = {
    "scene": (["costs", "labels", "seam", "patches", "leveling", "energy"], []),
    "labels": (["seam", "adjusted_patches", "patches", "leveling"], ["costs", "labels", "energy"]),
    "view_selection": (["seam", "adjusted_patches", "patches", "leveling"], ["costs", "labels", "energy"]),
    "rings": (["seam", "adjusted_patches"], ["costs", "labels", "patches", "energy"]),
    "adjacency": (["patches", "leveling", "energy"], ["costs", "labels", "seam"]),
    "undistort": (["costs", "energy", "seam", "patches", "leveling"], ["labels"]),
    "views": (["labels", "seam_run", "costs", "seam", "patches", "energy"], []),
    "face_range": (["costs", "energy"], ["labels", "seam", "patches"]),
}


@pytest.mark.parametrize("change", list(CASES))
@pytest.mark.parametrize("name", ["tiny", "occ"])
def test_a_changed_input_invalidates_what_is_derived_from_it(b2, scene_mod, get_scene, name, change):
    s = get_scene(name)
    smaller = scene_mod.sphere_scene(3, 6, 160, 120, axis_cams=True, name="tiny3")   # fewer faces than either
    assert smaller.faces.shape[0] < s.faces.shape[0]
    c = b2.Context(0)
    c.set_scene(s)
    _graph(c, scene_mod, s)
    before, (info, sinfo, pinfo) = _stages(c)

    probes = {
        "costs": lambda: c.data_costs_download(info.nnz),
        "labels": c.labels_download,
        "seam": lambda: c.seam_download(sinfo),
        "patches": lambda: c.texture_patches_download(pinfo),
        "leveling": c.local_seam_leveling_run,
        "energy": c.mrf_energy,
        "adjusted_patches": lambda: c.texture_patches_run(apply_adjust=True),
        "seam_run": c.seam_run,
    }
    expected = dict(costs=before["dc"], labels=before["labels"], seam=before["seam"], patches=before["patches"])

    scene, k, undistort = s, None, False
    if change == "scene":
        scene = smaller
        c.set_scene(scene)
    elif change == "labels":
        c.set_labels(before["labels"])
    elif change == "view_selection":
        c.view_selection_run()
    elif change == "rings":
        c.set_vertex_rings(*scene_mod.vertex_rings(s.faces, s.verts.shape[0]))
    elif change == "adjacency":
        c.set_adjacency(*scene_mod.face_adjacency(s.faces))
    elif change == "undistort":
        undistort = True
        c.undistort_views(*_distortion(s.num_views))
    elif change == "views":
        k = s.num_views - 1
        c.set_views(*_views(b2, s, k))
    elif change == "face_range":
        c.set_face_range(0, s.faces.shape[0])

    refused, kept = CASES[change]
    for p in kept:   # first: a refused stage run also discards its own earlier result
        got = probes[p]()
        if p in expected:
            assert _same(got, expected[p]), p
    for p in refused:
        with pytest.raises(b2.B2TexError) as e:
            probes[p]()
        assert e.value.rc == ARG and "missing or out of date" in str(e.value), (p, str(e.value))

    if change == "scene":
        _graph(c, scene_mod, scene)
    again, _ = _stages(c)
    c.close()
    assert _same(again, _fresh(b2, scene_mod, scene, k, undistort))
