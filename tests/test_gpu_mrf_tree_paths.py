"""-m gpu: every code path of the tree solver k_tree (csrc/mrf.cu) against the oracle, on synthetic view-selection inputs
built to select it:

* lanes per node G = 4, 8, 16 and 32, chosen by alloc_mrf from the candidates per face (16 both where it drops to 8
  because the launch has few trees, and where it stays 16);
* label lookup through bitmasks (K + 1 <= 2048, the last bit of the last word set) and by bisection (K >= 2048, up to the
  largest K = 65535);
* trees solved in shared memory, and trees solved through global memory because a label list is longer than the
  scratch (over 1024 labels, or longer than the scratch fits under the shared-memory limit for the group size) or a
  node has degree > 3 (a non-manifold fan);
* the plain, spanning-tree (k_tree<.., S>) and multilevel (weighted, k_tree<.., W>) schedules.

Costs lie on a 1/16 grid, so that many DP sums tie exactly: each lane-group reduction must break ties by the lowest
position, as the oracle does.  Every case checks the iterations, labels and fixed-point energy trace of the oracle's
schedule, and through b2tex_mrf_info the path it is named for, so that a tuning change cannot move a case elsewhere."""
import ctypes as C
import importlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TREE_WARPS = 16                  # warps of one k_tree block (TREE_THREADS / 32)
TREE_SMEM_MAX = 200 * 1024       # dynamic shared memory k_tree may use


def mask_words(K):
    """32-bit words of a label bitmask for labels 1 .. K, 0 where the kernel bisects the sorted label list instead"""
    w = (K + 1 + 31) // 32
    return 0 if K == 0 or w > 64 else w


def expected_tree_cap(G, mw, longest):
    """the longest label list of the input rounded up to 16 and at most 1024, lowered in steps of 16 until the
    scratch of all lane groups of a block fits the shared-memory limit"""
    cap = min(1024, max(16, (longest + 15) // 16 * 16))
    while cap > 16 and TREE_WARPS * (32 // G) * (cap * 6 + mw * 4 + ((mw * 2 + 3) & ~3)) > TREE_SMEM_MAX:
        cap -= 16
    return cap


# ---- seeded synthetic inputs ----------------------------------------------------------------------------------------
def grid_mesh(nx, ny, fan=0):
    """triangulated nx x ny grid in the plane (2 nx ny faces, every face degree <= 3); fan > 0 appends that many
    triangles on the diagonal of the middle cell, a non-manifold edge shared by fan + 2 faces"""
    i, j = np.meshgrid(np.arange(ny), np.arange(nx), indexing="ij")
    a = (i * (nx + 1) + j).ravel()
    b, c = a + 1, a + nx + 1
    d = c + 1
    faces = np.stack([np.stack([a, b, d], 1), np.stack([a, d, c], 1)], 1).reshape(-1, 3)
    vi, vj = np.meshgrid(np.arange(ny + 1), np.arange(nx + 1), indexing="ij")
    verts = np.stack([vj.ravel(), vi.ravel(), np.zeros(vi.size)], 1)
    mid = 2 * ((ny // 2) * nx + nx // 2)          # faces mid, mid + 1 share the diagonal (a, d) of the middle cell
    if fan:
        va, vd = faces[mid, 0], faces[mid, 2]
        apex = np.stack([verts[va] + [0.5, -0.5, 1.0 + k] for k in range(fan)])
        faces = np.concatenate([faces, np.stack([np.full(fan, va), np.full(fan, vd), len(verts) + np.arange(fan)], 1)])
        verts = np.concatenate([verts, apex])
    return verts.astype(np.float32), faces.astype(np.uint32), mid


def draw_views(rng, cnt, K):
    """per face cnt[f] distinct views in [0, K), ascending; CSR (face_ptr, view)"""
    F = len(cnt)
    small = cnt * 4 <= K
    fid = np.repeat(np.arange(F, dtype=np.int64), np.where(small, cnt + cnt // 2 + 8, 0))
    key = np.unique(fid * K + rng.integers(0, K, len(fid)))           # oversampled, duplicates dropped
    f = key // K
    order = np.lexsort((rng.random(len(key)), f))                     # a random subset of cnt[f] per face
    fo = f[order]
    rank = np.arange(len(fo)) - np.searchsorted(fo, np.arange(F))[fo]
    key = key[np.sort(order[rank < cnt[fo]])]
    ok = np.bincount(key // K, minlength=F) == cnt
    redo = np.flatnonzero(~ok)                                        # long lists, and short draws
    key = np.sort(np.concatenate([key[ok[key // K]]] + [r * K + rng.choice(K, cnt[r], replace=False) for r in redo]))
    assert np.array_equal(np.bincount(key // K, minlength=F), cnt)
    return np.concatenate([[0], np.cumsum(cnt)]).astype(np.uint64), (key % K).astype(np.uint16)


def tree_path_problem(seed, nx, ny, K, mean, hubs=(0, 0, 0, 0), last_view=False, full_face=False, fan=0,
                      continuous=False):
    """A view-selection input on a grid: candidate counts around `mean` (about 3 % of the faces unseen), `hubs` =
    (alone, pairs, lo, hi): that many hub faces on their own and pairs of adjacent hubs (parent and child both long)
    with lo .. hi candidates; last_view: the hubs and 1 % of the faces see view K - 1 at cost 0 (label K, the last
    bit of the bitmask); full_face: one face sees all K views; fan: a non-manifold fan whose faces and the two faces
    beside it are hubs; costs on a 1/16 grid unless continuous.  Returns a dict of the mesh, its adjacency and the
    DataCosts CSR."""
    scene = importlib.import_module("mvs-texturing_b200.scene")
    rng = np.random.default_rng(seed)
    verts, faces, mid = grid_mesh(nx, ny, fan)
    F = len(faces)
    ap, ai = scene.face_adjacency(faces)
    cnt = np.minimum(rng.poisson(mean - 1, F) + 1, K)
    cnt[rng.random(F) < 0.03] = 0
    alone, pairs, lo, hi = hubs
    pick = rng.permutation(F - fan)
    hub = list(pick[:alone]) + [w for f in pick[alone:alone + pairs] for w in (f, ai[ap[f]])]
    if fan:
        hub += [mid, mid + 1] + list(range(F - fan, F))
    hub = np.unique(np.asarray(hub, np.int64))
    cnt[hub] = rng.integers(lo, hi + 1, len(hub))
    if full_face:
        cnt[pick[-1]] = K
    fp, view = draw_views(rng, cnt, K)
    cost = (rng.random(len(view)) if continuous else rng.integers(0, 17, len(view)) / 16).astype(np.float32)
    if last_view:
        marked = np.union1d(hub, rng.choice(F, F // 100, replace=False))
        marked = marked[cnt[marked] > 0]
        view[fp[marked + 1] - 1] = K - 1                               # the largest view of the list: still ascending
        cost[fp[marked + 1] - 1] = 0.0
    return dict(verts=verts, faces=faces, ap=ap, ai=ai, fp=fp, view=view, cost=cost, K=K, F=F,
                longest=int(cnt.max()), rho=len(view) / F)


# name: generator arguments, G = the lanes per node alloc_mrf must choose; below: the scratch must be shorter than the
# longest list; degree4: a node of degree > 3; stay16: enough trees for G = 16 to stay 16 (root_div from the SM count)
CASES = {
    "g4": dict(gen=dict(nx=50, ny=50, K=40, mean=3, hubs=(4, 2, 20, 40)), G=4),
    "g8": dict(gen=dict(nx=50, ny=50, K=60, mean=8, hubs=(4, 2, 40, 60)), G=8),
    "g16_demoted": dict(gen=dict(nx=50, ny=50, K=100, mean=20, hubs=(4, 2, 60, 100)), G=8),
    "g16": dict(gen=dict(nx=100, ny=100, K=100, mean=20, hubs=(4, 2, 60, 100)), G=16, stay16=True),
    "g32": dict(gen=dict(nx=50, ny=50, K=200, mean=70, hubs=(4, 2, 150, 200)), G=32),
    "k2047_last_bit": dict(gen=dict(nx=50, ny=50, K=2047, mean=3, hubs=(4, 2, 100, 180), last_view=True), G=4),
    "k2048_no_masks": dict(gen=dict(nx=50, ny=50, K=2048, mean=8, hubs=(4, 2, 200, 400)), G=8),
    "k65535": dict(gen=dict(nx=50, ny=50, K=65535, mean=3, hubs=(4, 2, 150, 250), last_view=True), G=4),
    "over1024_g4": dict(gen=dict(nx=50, ny=50, K=3000, mean=3, hubs=(3, 2, 1025, 1500)), G=4, below=True),
    "over1024_g8": dict(gen=dict(nx=50, ny=50, K=3000, mean=8, hubs=(3, 2, 1025, 1500)), G=8, below=True),
    "over1024_g16": dict(gen=dict(nx=100, ny=100, K=3000, mean=18, hubs=(3, 2, 1025, 1500)), G=16, below=True,
                         stay16=True),
    "over1024_g32": dict(gen=dict(nx=50, ny=50, K=3000, mean=70, hubs=(3, 2, 1025, 1500)), G=32, below=True),
    # longer than the scratch of every lane group fits in TREE_SMEM_MAX
    "smem_g4_300": dict(gen=dict(nx=50, ny=50, K=300, mean=3, hubs=(3, 2, 300, 300)), G=4, below=True),
    "smem_g8_600": dict(gen=dict(nx=50, ny=50, K=1500, mean=8, hubs=(3, 2, 600, 600)), G=8, below=True),
    "smem_g16_1016": dict(gen=dict(nx=100, ny=100, K=1500, mean=18, hubs=(3, 2, 1016, 1016)), G=16, below=True,
                          stay16=True),
    "face_sees_all": dict(gen=dict(nx=50, ny=50, K=1000, mean=70, full_face=True), G=32),
    "fan_continuous": dict(gen=dict(nx=50, ny=50, K=300, mean=8, hubs=(0, 0, 200, 300), fan=3, continuous=True), G=8,
                           degree4=True),
}

_problems = {}


def problem(name):
    if name not in _problems:
        _problems[name] = tree_path_problem(sorted(CASES).index(name) + 11, **CASES[name]["gen"])
    return _problems[name]


@pytest.fixture(scope="module")
def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def schedules(orc):
    import oracle_multilevel as OM
    import oracle_spanning as OS
    OM.lib(); OS.lib()
    return dict(plain=(dict(), lambda *a, **kw: orc.view_selection(*a, threads=1, **kw)),
                spanning=(dict(use_spanning_tree=1), lambda *a, **kw: OS.view_selection(*a, **kw)),
                multilevel=(dict(use_multilevel=1), lambda *a, **kw: OM.view_selection(*a, use_multilevel=1, **kw)))


def mrf_kw(name, num_sms):
    """root_div of the case: one root candidate per root_div faces; stay16 keeps faces / root_div >= num_sms * 32"""
    if not CASES[name].get("stay16"):
        return {}
    F = problem(name)["F"]
    rd = F // (num_sms * 32)
    assert rd >= 1, "the mesh is too small for G = 16 on this device"
    return dict(root_div=rd)


_IMG = np.full((2, 2, 3), 128, np.uint8)


def resident(b2, pb):
    """a context holding the problem: the grid mesh, K 2 x 2 views (only K matters to view selection), the costs and
    the adjacency"""
    c = b2.Context(0)
    c.set_mesh(pb["verts"], pb["faces"], np.zeros((pb["F"], 3), np.float32))
    one = b2.B2View()
    one.width = one.height = 2
    one.rgb = _IMG.ctypes.data
    views = (b2.B2View * pb["K"])()
    C.memmove(views, bytes(one) * pb["K"], C.sizeof(views))
    c.set_views(views, pb["K"])
    c.set_data_costs(pb["fp"], pb["view"], pb["cost"])
    c.set_adjacency(pb["ap"], pb["ai"])
    return c


def check_path(info, name, schedule):
    """the info fields name the path the case is built for"""
    pb, case = problem(name), CASES[name]
    mw = mask_words(pb["K"])
    assert info.tree_group == case["G"]
    assert info.label_mask_words == mw
    assert info.tree_cap == expected_tree_cap(case["G"], mw, pb["longest"])
    assert TREE_WARPS * (32 // info.tree_group) * (info.tree_cap * 6 + mw * 4 + ((mw * 2 + 3) & ~3)) <= TREE_SMEM_MAX
    assert (info.tree_cap < pb["longest"]) == case.get("below", False)
    if case.get("below") or case.get("degree4"):
        assert info.global_trees > 0
    elif schedule != "multilevel":          # contracted graphs have nodes of any degree
        assert info.global_trees == 0


def check_oracle(info, trace, labels, o, schedule):
    assert info.iterations == o["iterations"]
    if schedule != "plain":
        assert info.multilevel_passes == o["multilevel_passes"] and info.coarse_nodes == o["coarse_nodes"]
    if schedule == "spanning":
        assert info.spanning_tree_iterations == o["spanning_tree_iterations"]
        assert info.spanning_tree_rejected == o["spanning_tree_rejected"]
    assert np.array_equal(trace, o["trace"])            # fixed-point energies of every iteration
    assert np.array_equal(labels, o["labels"])


@pytest.mark.parametrize("schedule", ["plain", "spanning", "multilevel"])
@pytest.mark.parametrize("name", list(CASES))
def test_tree_path_matches_oracle(b2, schedules, num_sms, name, schedule):
    pb = problem(name)
    kw = mrf_kw(name, num_sms)
    dev_kw, oracle = schedules[schedule]
    o = oracle(pb["ap"], pb["ai"], pb["fp"], pb["view"], pb["cost"], **kw)
    if CASES[name]["gen"].get("last_view"):
        assert (o["labels"] == pb["K"]).any()            # label K is chosen somewhere
    c = resident(b2, pb)
    info, trace = c.view_selection_run(**dev_kw, **kw)
    labels = c.labels_download()
    c.close()
    check_path(info, name, schedule)
    check_oracle(info, trace, labels, o, schedule)
    if schedule == "plain":   # the one-shot call: same labels, same path
        l1, i1 = b2.view_selection(b2.DataCosts(pb["F"], pb["K"], pb["fp"], pb["view"], pb["cost"]), pb["ap"], pb["ai"],
                                   **kw)
        assert np.array_equal(l1, labels) and i1.iterations == info.iterations
        assert (i1.tree_group, i1.tree_cap, i1.label_mask_words, i1.global_trees) == \
            (info.tree_group, info.tree_cap, info.label_mask_words, info.global_trees)


@pytest.mark.parametrize("name", ["smem_g4_300", "k2047_last_bit"])
def test_tree_path_two_parts(b2, orc, num_sms, name):
    """num_parts = 2: the multi-GPU schedule's partitioned forests on one device"""
    pb = problem(name)
    kw = dict(mrf_kw(name, num_sms), num_parts=2)
    o = orc.view_selection(pb["ap"], pb["ai"], pb["fp"], pb["view"], pb["cost"], threads=1, **kw)
    c = resident(b2, pb)
    info, trace = c.view_selection_run(**kw)
    labels = c.labels_download()
    c.close()
    check_path(info, name, "plain")
    check_oracle(info, trace, labels, o, "plain")


@pytest.mark.parametrize("name", ["tiny", "C2s", "C3s", "C5s"])
def test_scene_tree_cap_unchanged(b2, get_scene, oracle_pipeline, name):
    """on inputs whose scratch fits, the cap is the longest label list rounded up to 16 (at most 1024)"""
    s = get_scene(name)
    r = oracle_pipeline(name, ("dc", "mrf"))
    dc = r["dc"]
    labels, info = b2.view_selection(b2.DataCosts(s.num_faces, s.num_views, dc["face_ptr"], dc["view"], dc["cost"]),
                                     *r["adj"])
    longest = int(np.diff(dc["face_ptr"].astype(np.int64)).max())
    assert info.tree_cap == min(1024, (longest + 15) // 16 * 16)
    assert info.label_mask_words == mask_words(s.num_views)
    assert info.iterations == r["mrf"]["iterations"] and np.array_equal(labels, r["mrf"]["labels"])
