"""-m gpu: multilevel view selection (use_multilevel = 1, csrc/mrf_multilevel.cu) against the oracle schedule
(oracle/mrf_multilevel.c): the same labels, passes, coarse node count and fixed-point energy trace."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ml():
    import oracle_multilevel as OM
    OM.lib()
    return OM


def _oracle(ml, r):
    dc = r["dc"]
    if "ml" not in r:
        r["ml"] = ml.view_selection(r["adj"][0], r["adj"][1], dc["face_ptr"], dc["view"], dc["cost"], use_multilevel=1)
    return r["ml"]


def _resident(b2, s, r, **kw):
    dc = r["dc"]
    c = b2.Context(0)
    c.set_scene(s)
    c.set_data_costs(dc["face_ptr"], dc["view"], dc["cost"])
    c.set_adjacency(*r["adj"])
    return c


@pytest.mark.parametrize("name", ["tiny", "occ", "messy", "C2s", "C3s", "C5s"])
def test_multilevel_matches_oracle(b2, ml, get_scene, oracle_pipeline, name):
    s = get_scene(name)
    r = oracle_pipeline(name, ("dc", "mrf"))
    om = _oracle(ml, r)
    c = _resident(b2, s, r)
    info, trace = c.view_selection_run(use_multilevel=1)
    labels = c.labels_download()
    assert info.iterations == om["iterations"]
    assert info.multilevel_passes == om["multilevel_passes"]
    assert info.coarse_nodes == om["coarse_nodes"]
    assert np.array_equal(trace, om["trace"])        # fixed-point energies of every fine and coarse iteration
    assert np.array_equal(labels, om["labels"])
    # the default schedule is untouched by a multilevel run on the same context
    info0, trace0 = c.view_selection_run()
    assert info0.multilevel_passes == 0 and info0.coarse_nodes == 0
    assert info0.iterations == r["mrf"]["iterations"] and np.array_equal(c.labels_download(), r["mrf"]["labels"])
    c.close()


def test_one_shot_matches_resident(b2, ml, get_scene, oracle_pipeline):
    s = get_scene("C2s")
    r = oracle_pipeline("C2s", ("dc", "mrf"))
    dc = r["dc"]
    labels, info = b2.view_selection(b2.DataCosts(s.num_faces, s.num_views, dc["face_ptr"], dc["view"], dc["cost"]),
                                     *r["adj"], use_multilevel=1)
    om = _oracle(ml, r)
    assert info.multilevel_passes == om["multilevel_passes"] and info.iterations == om["iterations"]
    assert np.array_equal(labels, om["labels"])


def test_partitions_are_unsupported(b2, get_scene, oracle_pipeline):
    s = get_scene("occ")
    r = oracle_pipeline("occ", ("dc", "mrf"))
    c = _resident(b2, s, r)
    with pytest.raises(b2.B2TexError) as e:
        c.view_selection_run(use_multilevel=1, num_parts=2)
    assert e.value.rc == 5   # B2TEX_ERR_UNSUPPORTED
    info, _ = c.view_selection_run(num_parts=2)   # the context stays usable
    assert info.iterations >= 1
    c.close()


def test_triangle_soup_with_mostly_unseen_faces(b2, ml):
    """more faces than candidates and adjacency entries (no edges, 10 of 1000 faces seen): the contraction's per-face
    scratch must hold every face; labels, passes and node count as the oracle's"""
    F = 1000
    rng = np.random.default_rng(5)
    seen = np.zeros(F, bool)
    seen[rng.choice(F, 10, replace=False)] = True
    fp = np.concatenate([[0], np.cumsum(np.where(seen, 2, 0))]).astype(np.uint64)
    view = np.array(sum([sorted(rng.choice(6, 2, replace=False).tolist()) for _ in range(10)], []), np.uint16)
    cost = rng.random(len(view)).astype(np.float32)
    ap, ai = np.zeros(F + 1, np.uint32), np.zeros(0, np.uint32)
    om = ml.view_selection(ap, ai, fp, view, cost, use_multilevel=1)
    labels, info = b2.view_selection(b2.DataCosts(F, 6, fp, view, cost), ap, ai, use_multilevel=1)
    assert info.iterations == om["iterations"] and info.coarse_nodes == om["coarse_nodes"] == F
    assert info.multilevel_passes == om["multilevel_passes"]
    assert np.array_equal(labels, om["labels"])
