"""Spanning-tree view selection on the CPU oracle (oracle/mrf_spanning.c): the sampler's invariants, exactness on
tree-shaped problems, the acceptance rule, and the unchanged schedule with the flag off."""
import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

SCENES = ["tiny", "C1", "C1d", "C2s", "C3s", "occ", "messy", "C5s"]
NO_NODE = 0xFFFFFFFF
LVL_NONE, LVL_DEAD = 0xFFFFFFFF, 0xFFFFFFFE
SEED = 548923723


@pytest.fixture(scope="module")
def st():
    import oracle_spanning as OS
    OS.lib()
    return OS


def _mix32(x):
    x = np.asarray(x, np.uint64) & 0xFFFFFFFF
    x ^= x >> 16; x = (x * 0x7feb352d) & 0xFFFFFFFF
    x ^= x >> 15; x = (x * 0x846ca68b) & 0xFFFFFFFF
    x ^= x >> 16
    return x


def _prio(v, t, seed=SEED):
    seed_t = int(_mix32((seed + 0x9E3779B9 * (t + 1)) & 0xFFFFFFFF))
    return _mix32(np.asarray(v, np.uint64) ^ seed_t)


def path_rejection_mrf():
    """path 0-1-2-3, labels {1, 2} everywhere; the left half prefers 1, the right half 2, each by less than one Potts
    unit.  When the middle edge joins two trees, each tree switches to the other side's old label (the fixed neighbour
    pays for it), so the cut stays and both unaries rise: the iteration must be rejected."""
    ap = np.array([0, 1, 3, 5, 6], np.uint32)
    ai = np.array([1, 0, 2, 1, 3, 2], np.uint32)
    fp = np.arange(0, 10, 2, dtype=np.uint64)
    view = np.array([0, 1] * 4, np.uint16)
    cost = np.float32([0.0, 0.25, 0.0, 0.25, 0.25, 0.0, 0.25, 0.0])
    return ap, ai, fp, view, cost


def _argmin_start(fp, view, cost):
    fp = fp.astype(np.int64)
    return np.array([view[fp[i] + np.argmin(cost[fp[i]:fp[i + 1]])] + 1 if fp[i + 1] > fp[i] else 0
                     for i in range(len(fp) - 1)], np.uint32)


def _tree_of(parent, v):
    while parent[v] != NO_NODE:
        v = parent[v]
    return v


def rejection_iteration(st):
    """the first iteration whose spanning forest of path_rejection_mrf cuts the middle edge"""
    ap, ai, fp, _, _ = path_rejection_mrf()
    for t in range(1, 200):
        _, parent, _ = st.sample_spanning(ap, ai, fp, t)
        if _tree_of(parent, 1) != _tree_of(parent, 2):
            return t
    raise AssertionError("no iteration splits the path")


@pytest.mark.parametrize("name", SCENES)
def test_sampler_invariants(orc, st, oracle_pipeline, name):
    r = oracle_pipeline(name, ("dc", "mrf"))
    ap, ai = r["adj"]
    fp = r["dc"]["face_ptr"]
    F = len(fp) - 1
    seen = np.diff(fp.astype(np.int64)) > 0
    src = np.repeat(np.arange(F), np.diff(ap.astype(np.int64)))
    keep = seen[src] & seen[ai]
    _, comp = connected_components(sp.csr_matrix((np.ones(int(keep.sum())), (src[keep], ai[keep])), shape=(F, F)),
                                   directed=False)
    for t in (1, 2, 7):
        for root_div in (64, 0):
            level, parent, depth = st.sample_spanning(ap, ai, fp, t, root_div=root_div)
            assert depth < 1022
            acyclic = orc.mrf_sample_forest(ap, ai, fp, t, root_div=root_div)
            roots = level == 0
            assert np.array_equal(roots, acyclic == 0)
            assert np.all(level[~seen] == LVL_DEAD) and np.all(parent[~seen] == NO_NODE)
            reached = level <= depth
            assert np.all(parent[roots] == NO_NODE)
            # every seen node of a component that holds a root is reached, nothing else is
            rooted = np.zeros(comp.max() + 1, bool)
            rooted[comp[roots]] = True
            assert np.array_equal(reached, seen & rooted[comp])
            assert np.all(level[seen & ~reached] == LVL_NONE)
            # one parent per reached non-root, one level up, the strongest neighbour at that level
            kids = np.flatnonzero(reached & ~roots)
            assert int(np.sum(parent != NO_NODE)) == int(reached.sum()) - int(roots.sum())
            assert np.all(level[parent[kids]] == level[kids] - 1)
            pr = _prio(np.arange(F), t)
            for v in kids[:: max(1, len(kids) // 2000)]:
                nb = ai[ap[v]:ap[v + 1]]
                up = nb[level[nb] == level[v] - 1]
                assert parent[v] == up[np.argmax(pr[up])]


def _random_tree(rng, n, K, maxl):
    nb = [[] for _ in range(n)]
    for v in range(1, n):
        u = int(rng.integers(0, v))
        nb[u].append(v); nb[v].append(u)
    ap = np.concatenate([[0], np.cumsum([len(x) for x in nb])]).astype(np.uint32)
    ai = np.array(sum([sorted(x) for x in nb], []), np.uint32)
    lists = [sorted(rng.choice(K, int(rng.integers(1, maxl + 1)), replace=False).tolist()) for _ in range(n)]
    fp = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.uint64)
    return ap, ai, fp, np.array(sum(lists, []), np.uint16), rng.random(sum(map(len, lists))).astype(np.float32)


def test_exact_on_trees(orc, st):
    """root_div = 0 on a tree-shaped MRF: one spanning tree covers it and has no non-tree edge, so the first iteration
    from the arg-min start reaches the exhaustive minimum"""
    rng = np.random.default_rng(17)
    for _ in range(40):
        n = int(rng.integers(2, 11))
        ap, ai, fp, view, cost = _random_tree(rng, n, 4, 3)
        best, _ = orc.mrf_brute_force(ap, ai, fp, view, cost)
        start = _argmin_start(fp, view, cost)
        it = st.spanning_iteration(ap, ai, fp, view, cost, start, 1, root_div=0)
        assert not it["rejected"]
        assert np.all(it["level"] <= n)
        e = orc.mrf_energy_fixed(ap, ai, fp, view, cost, it["labels"]) / 2.0 ** 32
        assert abs(e - best) <= 1e-5


def test_rejection_restores_the_labels(orc, st):
    ap, ai, fp, view, cost = path_rejection_mrf()
    t = rejection_iteration(st)
    start = np.array([1, 1, 2, 2], np.uint32)
    it = st.spanning_iteration(ap, ai, fp, view, cost, start, t)
    assert list(it["swept"]) == [2, 2, 1, 1]
    assert it["rejected"] and np.array_equal(it["labels"], start)
    e0 = orc.mrf_energy_fixed(ap, ai, fp, view, cost, start)
    assert orc.mrf_energy_fixed(ap, ai, fp, view, cost, it["swept"]) > e0
    # the schedule: that iteration keeps the labels and the energy of the one before
    run = st.view_selection(ap, ai, fp, view, cost, max_iterations=t)
    assert run["spanning_tree_rejected"] >= 1
    assert np.all(np.diff(run["trace"]) <= 0)


@pytest.mark.parametrize("name", [s for s in SCENES if s != "C5s"])   # C5s: the GPU test compares it with the device
def test_schedule(orc, st, oracle_pipeline, name):
    import oracle_multilevel as OM
    r = oracle_pipeline(name, ("dc", "mrf"))
    dc, off = r["dc"], r["mrf"]
    ap, ai = r["adj"]
    args = (ap, ai, dc["face_ptr"], dc["view"], dc["cost"])
    on = st.view_selection(*args)
    assert np.all(np.diff(on["trace"]) <= 0)
    assert 1 <= on["spanning_tree_iterations"] <= on["iterations"]
    assert on["spanning_tree_rejected"] <= on["spanning_tree_iterations"]
    assert on["iterations"] == on["spanning_tree_iterations"] + on["acyclic_iterations"]
    assert on["trace"][-1] == orc.mrf_energy_fixed(*args, on["labels"]) / 2.0 ** 32
    # the spanning phase iteration by iteration: a rejected iteration leaves exactly the labels before it
    labels = _argmin_start(dc["face_ptr"], dc["view"], dc["cost"])
    for t in range(1, min(on["spanning_tree_iterations"], 4) + 1):
        it = st.spanning_iteration(*args, labels, t)
        if it["rejected"]:
            assert np.array_equal(it["labels"], labels)
        else:
            assert np.array_equal(it["labels"], it["swept"])
        labels = it["labels"]
        assert orc.mrf_energy_fixed(*args, labels) / 2.0 ** 32 == on["trace"][t]
    # with multilevel as well
    both = st.view_selection(*args, use_multilevel=1)
    assert both["spanning_tree_iterations"] == on["spanning_tree_iterations"]
    assert np.array_equal(both["trace"][:on["spanning_tree_iterations"] + 1], on["trace"][:on["spanning_tree_iterations"] + 1])
    assert np.all(np.diff(both["trace"]) <= 0)
    # flag off: exactly the existing schedules
    same = st.view_selection(*args, use_spanning_tree=0)
    assert same["iterations"] == off["iterations"] and np.array_equal(same["labels"], off["labels"])
    assert np.array_equal(same["trace"], off["trace"]) and same["spanning_tree_iterations"] == 0
    ml = OM.view_selection(*args, use_multilevel=1)
    same = st.view_selection(*args, use_spanning_tree=0, use_multilevel=1)
    assert same["iterations"] == ml["iterations"] and same["multilevel_passes"] == ml["multilevel_passes"]
    assert same["coarse_nodes"] == ml["coarse_nodes"]
    assert np.array_equal(same["labels"], ml["labels"]) and np.array_equal(same["trace"], ml["trace"])
