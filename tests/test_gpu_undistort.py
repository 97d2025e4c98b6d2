"""-m gpu: undistortion of the resident views (b2tex_undistort_views, k_undistort) against the oracle's restatement (oracle/undistort.c), and
every later stage on undistorted views against the same stages on images undistorted beforehand."""
import numpy as np
import pytest

import oracle_undistort as ou   # oracle/ is on sys.path (tests/conftest.py)

pytestmark = pytest.mark.gpu

# per view (flen, k0, k1): pincushion in both models (k2 > 0 for Bundler's, k < 0 for VisualSFM's): the undistorted
# images have black corners, so every view gets a validity mask
PINCUSHION = [(0.9, 0.12, 0.03), (1.0, -0.15, 0.0), (0.8, 0.1, 0.05)]


def _rgb(b2, c, s):
    import torch
    from importlib import import_module
    ptr, n = c.device_ptr("rgb")
    K, H, W = s.num_views, s.height, s.width
    assert n >= 3 * K * H * W
    par = import_module("mvs-texturing_b200.sharded")
    return torch.as_tensor(par._DevArray(ptr, 3 * K * H * W, "|u1"), device="cuda").cpu().numpy().reshape(K, H, W, 3)


def _coeffs(K, table):
    flen = np.array([table[v % len(table)][0] for v in range(K)], np.float32)
    dist = np.array([table[v % len(table)][1:] for v in range(K)], np.float32)
    return flen, dist


def test_undistorted_images_bit_exact(b2, get_scene, orc):
    """mixed per-view coefficients: both models, black borders and none, a VisualSFM view without a root in its corners,
    and views left alone (k0 == 0, also with k1 != 0)"""
    s = get_scene("small")
    table = [(0.9, 0.12, 0.03), (0.5, -0.9, 0.0), (1.0, 0.0, 0.2), (1.1, -0.05, 0.0), (0.8, 0.2, 0.0), (1.0, 0.0, 0.0)]
    flen, dist = _coeffs(s.num_views, table)
    c = b2.Context(0)
    c.set_scene(s)
    c.undistort_views(flen, dist)
    g = _rgb(b2, c, s)
    c.close()
    for v in range(s.num_views):
        ref = ou.undistort(s.images[v], flen[v], dist[v, 0], dist[v, 1])
        assert np.array_equal(g[v], ref), (v, int((g[v] != ref).any(-1).sum()))
        if dist[v, 0] == 0:
            assert np.array_equal(g[v], s.images[v])


def _all_stages(b2, scene_mod, s, images=None, undistort=None):
    c = b2.Context(0)
    c.set_scene(s, images)
    if undistort is not None:
        c.undistort_views(*undistort)
    c.set_adjacency(*scene_mod.face_adjacency(s.faces))
    c.set_vertex_rings(*scene_mod.vertex_rings(s.faces, s.verts.shape[0]))
    info = c.data_costs_run()
    out = dict(dc=c.data_costs_download(info.nnz, quality=True))
    c.view_selection_run()
    out["labels"] = c.labels_download()
    sinfo = c.seam_run()
    out["seam"] = c.seam_download(sinfo)
    pinfo = c.texture_patches_run(apply_adjust=True)
    c.local_seam_leveling_run()
    out["patches"] = c.texture_patches_download(pinfo)
    c.close()
    return out


def _same(a, b):
    assert set(a["dc"]) == set(b["dc"])
    for k in ("face_ptr", "view", "cost", "quality"):
        assert np.array_equal(a["dc"][k].view(np.uint8), b["dc"][k].view(np.uint8)), k
    assert np.array_equal(a["labels"], b["labels"])
    for k in ("row_ptr", "row_label", "x"):
        assert np.array_equal(a["seam"][k].view(np.uint8), b["seam"][k].view(np.uint8)), k
    assert len(a["patches"]) == len(b["patches"]) > 0
    for p, q in zip(a["patches"], b["patches"]):
        for k in ("label", "min_x", "min_y", "faces"):
            assert p[k] == q[k], k
        for k in ("texcoords", "image", "validity", "blending"):
            assert np.array_equal(p[k].view(np.uint8), q[k].view(np.uint8)), k


def test_every_stage_reads_the_undistorted_pixels(b2, get_scene, scene_mod, orc):
    """`occ` (real occlusion) with a pincushion distortion on every view: undistorting on the device and uploading images
    undistorted beforehand give byte-identical data costs, labels, adjust values, patches and masks; the data costs and
    labels are those of the oracle on the undistorted images."""
    s = get_scene("occ")
    flen, dist = _coeffs(s.num_views, PINCUSHION)
    und = np.stack([ou.undistort(s.images[v], flen[v], dist[v, 0], dist[v, 1]) for v in range(s.num_views)])
    assert all((und[v][[0, 0, -1, -1], [0, -1, 0, -1]] == 0).all(-1).any() for v in range(s.num_views))   # all flagged
    a = _all_stages(b2, scene_mod, s, undistort=(flen, dist))
    b = _all_stages(b2, scene_mod, s, images=und)
    _same(a, b)
    o = orc.data_costs(s, images=und)
    assert np.array_equal(a["dc"]["face_ptr"], o["face_ptr"]) and np.array_equal(a["dc"]["view"], o["view"])
    assert np.array_equal(a["dc"]["quality"].view(np.uint32), o["quality"].view(np.uint32))
    assert np.array_equal(a["dc"]["cost"].view(np.uint32), o["cost"].view(np.uint32))
    ap, ai = scene_mod.face_adjacency(s.faces)
    om = orc.view_selection(ap, ai, o["face_ptr"], o["view"], o["cost"], threads=1)
    assert np.array_equal(a["labels"], om["labels"])
    plain = _all_stages(b2, scene_mod, s)
    assert not np.array_equal(plain["dc"]["cost"], a["dc"]["cost"])   # the distortion does change the result


def test_zero_distortion_changes_nothing(b2, get_scene, scene_mod):
    s = get_scene("occ")
    K = s.num_views
    flen = np.full(K, 0.9, np.float32)
    dist = np.zeros((K, 2), np.float32)
    dist[::2, 1] = 0.3   # k1 alone does not select undistortion (generate_texture_views.cpp:154)
    _same(_all_stages(b2, scene_mod, s, undistort=(flen, dist)), _all_stages(b2, scene_mod, s))


def test_argument_errors(b2, get_scene):
    s = get_scene("tiny")
    K = s.num_views
    c = b2.Context(0)
    with pytest.raises(b2.B2TexError) as e:   # no views set
        c.undistort_views(np.ones(K, np.float32), np.full((K, 2), 0.1, np.float32))
    assert e.value.rc == 3
    c.set_scene(s)
    bad = [(np.ones(K - 1, np.float32), np.full((K - 1, 2), 0.1, np.float32)),                   # wrong count
           (np.array([1.0] * (K - 1) + [0.0], np.float32), np.full((K, 2), 0.1, np.float32)),     # flen 0
           (np.array([np.nan] + [1.0] * (K - 1), np.float32), np.full((K, 2), 0.1, np.float32)),  # flen NaN
           (np.array([-1.0] + [1.0] * (K - 1), np.float32), np.full((K, 2), 0.1, np.float32)),    # flen < 0
           (np.array([np.inf] + [1.0] * (K - 1), np.float32), np.full((K, 2), 0.1, np.float32))]  # flen inf
    before = _rgb(b2, c, s)
    for flen, dist in bad:
        with pytest.raises(b2.B2TexError) as e:
            c.undistort_views(flen, dist)
        assert e.value.rc == 3
    assert np.array_equal(_rgb(b2, c, s), before)   # a rejected call touches no pixel
    dist = np.zeros((K, 2), np.float32)
    dist[1, 0] = 0.1
    c.undistort_views(np.array([0.0, 1.0] + [-5.0] * (K - 2), np.float32), dist)   # flen of untouched views is not read
    c.close()
