"""-m gpu: spanning-tree view selection (use_spanning_tree = 1, csrc/mrf.cu's k_forest<true> / k_tree_prep<true> /
k_accept / k_restore) against the oracle schedule (oracle/mrf_spanning.c): the same labels, iterations per phase,
rejected iterations and fixed-point energy trace, alone and together with the multilevel schedule."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def st():
    import oracle_spanning as OS
    OS.lib()
    return OS


def _oracle(st, r, use_multilevel=0):
    dc = r["dc"]
    key = ("st", use_multilevel)
    if key not in r:
        r[key] = st.view_selection(r["adj"][0], r["adj"][1], dc["face_ptr"], dc["view"], dc["cost"],
                                   use_multilevel=use_multilevel)
    return r[key]


def _resident(b2, s, r):
    dc = r["dc"]
    c = b2.Context(0)
    c.set_scene(s)
    c.set_data_costs(dc["face_ptr"], dc["view"], dc["cost"])
    c.set_adjacency(*r["adj"])
    return c


def _check(c, o, use_multilevel):
    info, trace = c.view_selection_run(use_spanning_tree=1, use_multilevel=use_multilevel)
    labels = c.labels_download()
    assert info.iterations == o["iterations"]
    assert info.spanning_tree_iterations == o["spanning_tree_iterations"]
    assert info.spanning_tree_rejected == o["spanning_tree_rejected"]
    assert info.multilevel_passes == o["multilevel_passes"] and info.coarse_nodes == o["coarse_nodes"]
    assert np.array_equal(trace, o["trace"])        # fixed-point energies of every iteration, rejected ones included
    assert np.array_equal(labels, o["labels"])


@pytest.mark.parametrize("name,use_multilevel", [(n, 0) for n in ("tiny", "occ", "messy", "C2s", "C3s", "C5s")]
                         + [(n, 1) for n in ("C2s", "C3s")])
def test_spanning_tree_matches_oracle(b2, st, get_scene, oracle_pipeline, name, use_multilevel):
    s = get_scene(name)
    r = oracle_pipeline(name, ("dc", "mrf"))
    c = _resident(b2, s, r)
    _check(c, _oracle(st, r, use_multilevel), use_multilevel)
    # the default schedule is untouched by a spanning-tree run on the same context
    info0, trace0 = c.view_selection_run()
    assert info0.spanning_tree_iterations == 0 and info0.spanning_tree_rejected == 0 and info0.multilevel_passes == 0
    assert info0.iterations == r["mrf"]["iterations"] and np.array_equal(c.labels_download(), r["mrf"]["labels"])
    assert np.array_equal(trace0, r["mrf"]["trace"])
    c.close()


def test_one_shot_matches_resident(b2, st, get_scene, oracle_pipeline):
    s = get_scene("C2s")
    r = oracle_pipeline("C2s", ("dc", "mrf"))
    dc = r["dc"]
    labels, info = b2.view_selection(b2.DataCosts(s.num_faces, s.num_views, dc["face_ptr"], dc["view"], dc["cost"]),
                                     *r["adj"], use_spanning_tree=1)
    o = _oracle(st, r)
    assert info.iterations == o["iterations"] and info.spanning_tree_iterations == o["spanning_tree_iterations"]
    assert info.spanning_tree_rejected == o["spanning_tree_rejected"]
    assert np.array_equal(labels, o["labels"])


def test_partitions_are_unsupported(b2, get_scene, oracle_pipeline):
    s = get_scene("occ")
    r = oracle_pipeline("occ", ("dc", "mrf"))
    c = _resident(b2, s, r)
    with pytest.raises(b2.B2TexError) as e:
        c.view_selection_run(use_spanning_tree=1, num_parts=2)
    assert e.value.rc == 5   # B2TEX_ERR_UNSUPPORTED
    assert "spanning-tree" in str(e.value)
    info, _ = c.view_selection_run(num_parts=2)   # the context stays usable
    assert info.iterations >= 1
    c.close()


def test_rejected_iterations_on_the_device(b2, st):
    """the path MRF whose middle edge joins two trees: the device undoes the same iterations as the oracle"""
    from test_mrf_spanning_cpu import path_rejection_mrf
    ap, ai, fp, view, cost = path_rejection_mrf()
    o = st.view_selection(ap, ai, fp, view, cost)
    labels, info = b2.view_selection(b2.DataCosts(4, 2, fp, view, cost), ap, ai, use_spanning_tree=1)
    assert o["spanning_tree_rejected"] >= 1
    assert info.spanning_tree_rejected == o["spanning_tree_rejected"]
    assert info.iterations == o["iterations"] and info.spanning_tree_iterations == o["spanning_tree_iterations"]
    assert np.array_equal(labels, o["labels"])


def test_triangle_soup_with_mostly_unseen_faces(b2, st):
    """no edges, 10 of 1000 faces seen: every seen face is a root, the spanning forest has no edges"""
    F = 1000
    rng = np.random.default_rng(5)
    seen = np.zeros(F, bool)
    seen[rng.choice(F, 10, replace=False)] = True
    fp = np.concatenate([[0], np.cumsum(np.where(seen, 2, 0))]).astype(np.uint64)
    view = np.array(sum([sorted(rng.choice(6, 2, replace=False).tolist()) for _ in range(10)], []), np.uint16)
    cost = rng.random(len(view)).astype(np.float32)
    ap, ai = np.zeros(F + 1, np.uint32), np.zeros(0, np.uint32)
    for use_multilevel in (0, 1):
        o = st.view_selection(ap, ai, fp, view, cost, use_multilevel=use_multilevel)
        labels, info = b2.view_selection(b2.DataCosts(F, 6, fp, view, cost), ap, ai, use_spanning_tree=1,
                                         use_multilevel=use_multilevel)
        assert info.iterations == o["iterations"] and info.spanning_tree_iterations == o["spanning_tree_iterations"]
        assert info.spanning_tree_rejected == o["spanning_tree_rejected"] == 0
        assert info.multilevel_passes == o["multilevel_passes"]
        assert np.array_equal(labels, o["labels"])
