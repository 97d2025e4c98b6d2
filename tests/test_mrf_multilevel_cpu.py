"""Multilevel view selection on the CPU oracle (oracle/mrf_multilevel.c): the schedule's invariants, the contraction's
exact energy identity, and a bound against exhaustive search on small random problems."""
import numpy as np
import pytest

SCENES = ["tiny", "C1", "C1d", "C2s", "C3s", "occ", "messy", "C5s"]


@pytest.fixture(scope="module")
def ml():
    import oracle_multilevel as OM
    OM.lib()
    return OM


@pytest.mark.parametrize("name", SCENES)
def test_schedule_invariants(orc, ml, oracle_pipeline, name):
    r = oracle_pipeline(name, ("dc", "mrf"))
    dc, off = r["dc"], r["mrf"]
    ap, ai = r["adj"]
    on = ml.view_selection(ap, ai, dc["face_ptr"], dc["view"], dc["cost"], use_multilevel=1)
    # the first fine phase is the default run, label for label and energy for energy
    assert on["first_phase_iterations"] == off["iterations"]
    assert np.array_equal(on["first_labels"], off["labels"])
    assert np.array_equal(on["trace"][:off["iterations"] + 1], off["trace"])
    # fine, coarse and later fine iterations never raise the energy
    assert np.all(np.diff(on["trace"]) <= 0)
    assert on["contractions"] >= 1 and on["identity_failures"] == 0
    assert on["multilevel_passes"] <= on["contractions"] <= on["multilevel_passes"] + 1
    e_off = orc.mrf_energy_fixed(ap, ai, dc["face_ptr"], dc["view"], dc["cost"], off["labels"])
    e_on = orc.mrf_energy_fixed(ap, ai, dc["face_ptr"], dc["view"], dc["cost"], on["labels"])
    assert e_on <= e_off
    assert (e_on < e_off) == (on["multilevel_passes"] > 0)
    assert on["trace"][-1] == e_on / 2.0 ** 32
    # flag off: exactly orc_view_selection
    same = ml.view_selection(ap, ai, dc["face_ptr"], dc["view"], dc["cost"], use_multilevel=0)
    assert same["iterations"] == off["iterations"] and np.array_equal(same["labels"], off["labels"])


@pytest.mark.parametrize("name", ["occ", "messy", "C2s"])
def test_contraction_energy_identity_on_random_labelings(orc, ml, oracle_pipeline, name):
    """fine energy of a labeling == coarse energy of its contraction (+ one per unseen face), in 32.32 fixed point"""
    r = oracle_pipeline(name, ("dc", "mrf"))
    dc = r["dc"]
    ap, ai = r["adj"]
    fp, view, cost = dc["face_ptr"].astype(np.int64), dc["view"], dc["cost"]
    rng = np.random.default_rng(7)
    n = np.diff(fp)
    for blocky in (False, True):
        pick = rng.integers(0, np.maximum(n, 1))
        if blocky:   # mostly the lowest label: large regions
            pick[rng.random(len(n)) < 0.8] = 0
        labels = np.where(n > 0, view[np.minimum(fp[:-1] + pick, max(len(view) - 1, 0))].astype(np.uint32) + 1, 0)
        labels = labels.astype(np.uint32)
        c = ml.contract(ap, ai, dc["face_ptr"], view, cost, labels)
        assert c["energy_fixed"] == orc.mrf_energy_fixed(ap, ai, dc["face_ptr"], view, cost, labels)
        assert np.array_equal(c["labels"][c["region"]], labels)
        assert c["size"].sum() == len(labels) and np.array_equal(np.bincount(c["region"], minlength=c["num_nodes"]), c["size"])
        # nodes are numbered by their lowest face
        first = np.full(c["num_nodes"], len(labels))
        np.minimum.at(first, c["region"], np.arange(len(labels)))
        assert np.all(np.diff(first) > 0)
        # symmetric weights, sum = fine adjacency entries that cross nodes
        cross = int(np.sum(c["region"][np.repeat(np.arange(len(labels)), np.diff(ap))] != c["region"][ai]))
        assert c["weight"].sum() == cross
        W = {}
        for a in range(c["num_nodes"]):
            for k in range(c["adj_ptr"][a], c["adj_ptr"][a + 1]):
                W[(a, int(c["adj_idx"][k]))] = c["weight"][k]
        assert all(W[(b, a)] == w for (a, b), w in W.items())


def test_contraction_by_hand(ml):
    """path 0-1-2-3-4, labels 1 1 2 2 1: nodes {0,1} {2,3} {4}; lists are intersections, costs sums in face order"""
    ap = np.array([0, 1, 3, 5, 7, 8], np.uint32)
    ai = np.array([1, 0, 2, 1, 3, 2, 4, 3], np.uint32)
    lists = [[0, 1], [0, 1, 2], [1], [0, 1], [0, 2]]
    costs = [[0.25, 0.5], [0.125, 0.75, 0.0], [0.5], [0.375, 0.0625], [0.0, 1.0]]
    fp = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.uint64)
    view = np.array(sum(lists, []), np.uint16)
    cost = np.array(sum(costs, []), np.float32)
    c = ml.contract(ap, ai, fp, view, cost, np.array([1, 1, 2, 2, 1], np.uint32))
    assert c["num_nodes"] == 3
    assert list(c["region"]) == [0, 0, 1, 1, 2] and list(c["labels"]) == [1, 2, 1] and list(c["size"]) == [2, 2, 1]
    assert list(c["ptr"]) == [0, 2, 3, 5]
    assert list(c["view"]) == [0, 1, 1, 0, 2]
    assert np.array_equal(c["cost"], np.float32([0.375, 1.25, 0.5625, 0.0, 1.0]))
    assert list(c["adj_ptr"]) == [0, 1, 3, 4] and list(c["adj_idx"]) == [1, 0, 2, 1]
    assert list(c["weight"]) == [1.0, 1.0, 1.0, 1.0]


def _random_problem(rng, n, K, maxl):
    edges = set()
    for v in range(1, n):   # a random tree plus extra edges: loops
        edges.add((int(rng.integers(0, v)), v))
    for _ in range(n // 2):
        a, b = sorted(rng.choice(n, 2, replace=False).tolist())
        edges.add((a, b))
    nb = [[] for _ in range(n)]
    for a, b in edges:
        nb[a].append(b); nb[b].append(a)
    ap = np.concatenate([[0], np.cumsum([len(x) for x in nb])]).astype(np.uint32)
    ai = np.array(sum([sorted(x) for x in nb], []), np.uint32)
    lists = [sorted(rng.choice(K, int(rng.integers(1, maxl + 1)), replace=False).tolist()) for _ in range(n)]
    fp = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.uint64)
    view = np.array(sum(lists, []), np.uint16)
    cost = rng.random(len(view)).astype(np.float32)
    return ap, ai, fp, view, cost


def test_bounded_by_exhaustive_search(orc, ml):
    """the exhaustive minimum is only reachable for ~10 nodes (tiny's 320 faces are far beyond it): 40 random problems,
    trees plus extra edges (loops), up to 3 of 4 labels per node"""
    rng = np.random.default_rng(3)
    for _ in range(40):
        ap, ai, fp, view, cost = _random_problem(rng, 10, 4, 3)
        best, _ = orc.mrf_brute_force(ap, ai, fp, view, cost)
        off = orc.view_selection(ap, ai, fp, view, cost, threads=1)
        on = ml.view_selection(ap, ai, fp, view, cost, use_multilevel=1)
        assert on["identity_failures"] == 0
        assert best - 1e-5 <= on["energy"] <= off["energy"] + 1e-9
