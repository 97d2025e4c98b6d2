"""-m gpu: texrecon's mapMAP schedule (spanning_tree_multilevel_after_n_iterations = n, csrc/mrf.cu's
enqueue_multilevel_step) against the oracle schedule (oracle/mrf_mapmap.c): the same labels, iterations per phase,
multilevel steps, rejections and fixed-point energy trace."""
import numpy as np
import pytest

from test_mrf_mapmap_cpu import step_rejection_mrf

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mm():
    import oracle_mapmap as OM
    OM.lib()
    return OM


def _resident(b2, s, r):
    dc = r["dc"]
    c = b2.Context(0)
    c.set_scene(s)
    c.set_data_costs(dc["face_ptr"], dc["view"], dc["cost"])
    c.set_adjacency(*r["adj"])
    return c


def _oracle(mm, r, n):
    key = ("mapmap", n)
    if key not in r:
        dc = r["dc"]
        r[key] = mm.view_selection(r["adj"][0], r["adj"][1], dc["face_ptr"], dc["view"], dc["cost"], n=n)
    return r[key]


def _same(info, o):
    assert info.iterations == o["iterations"]
    assert info.spanning_tree_iterations == o["spanning_tree_iterations"]
    assert info.spanning_tree_rejected == o["spanning_tree_rejected"]
    assert info.multilevel_steps == o["multilevel_steps"]
    assert info.multilevel_steps_rejected == o["multilevel_steps_rejected"]
    assert info.coarse_nodes == o["coarse_nodes"] and info.multilevel_passes == 0


@pytest.mark.parametrize("name,n", [(s, 5) for s in ("tiny", "occ", "messy", "C2s", "C3s", "C5s")] + [("C2s", 1), ("C2s", 3)])
def test_mapmap_matches_oracle(b2, mm, get_scene, oracle_pipeline, name, n):
    s = get_scene(name)
    r = oracle_pipeline(name, ("dc", "mrf"))
    o = _oracle(mm, r, n)
    c = _resident(b2, s, r)
    info, trace = c.view_selection_run(use_spanning_tree=1, use_multilevel=1, spanning_tree_multilevel_after_n_iterations=n)
    _same(info, o)
    assert np.array_equal(trace, o["trace"])        # fixed-point energies of every iteration, steps included
    assert np.array_equal(c.labels_download(), o["labels"])
    # the default schedule is untouched by such a run on the same context
    info0, trace0 = c.view_selection_run()
    assert info0.multilevel_steps == 0 and info0.spanning_tree_iterations == 0 and info0.multilevel_passes == 0
    assert info0.iterations == r["mrf"]["iterations"] and np.array_equal(c.labels_download(), r["mrf"]["labels"])
    assert np.array_equal(trace0, r["mrf"]["trace"])
    c.close()


def test_one_shot_matches_oracle(b2, mm, get_scene, oracle_pipeline):
    s = get_scene("C2s")
    r = oracle_pipeline("C2s", ("dc", "mrf"))
    dc = r["dc"]
    p = b2.texrecon_mrf_params()
    kw = {k: getattr(p, k) for k in ("use_spanning_tree", "use_multilevel", "spanning_tree_multilevel_after_n_iterations")}
    labels, info = b2.view_selection(b2.DataCosts(s.num_faces, s.num_views, dc["face_ptr"], dc["view"], dc["cost"]),
                                     *r["adj"], **kw)
    o = _oracle(mm, r, 5)
    _same(info, o)
    assert np.array_equal(labels, o["labels"])


def test_rejected_step_on_the_device(b2, mm):
    ap, ai, fp, view, cost = step_rejection_mrf()
    o = mm.view_selection(ap, ai, fp, view, cost, n=1, max_iterations=12)
    assert o["multilevel_steps_rejected"] >= 1
    labels, info = b2.view_selection(b2.DataCosts(7, 2, fp, view, cost), ap, ai, use_spanning_tree=1, use_multilevel=1,
                                     spanning_tree_multilevel_after_n_iterations=1, max_iterations=12)
    _same(info, o)
    assert np.array_equal(labels, o["labels"])


def test_errors_leave_the_context_usable(b2, get_scene, oracle_pipeline):
    s = get_scene("occ")
    r = oracle_pipeline("occ", ("dc", "mrf"))
    c = _resident(b2, s, r)
    for flags in (dict(use_spanning_tree=1), dict(use_multilevel=1), {}):
        with pytest.raises(b2.B2TexError) as e:
            c.view_selection_run(spanning_tree_multilevel_after_n_iterations=5, **flags)
        assert e.value.rc == 3   # B2TEX_ERR_ARG
        assert "spanning_tree_multilevel_after_n_iterations" in str(e.value)
    with pytest.raises(b2.B2TexError) as e:
        c.view_selection_run(use_spanning_tree=1, use_multilevel=1, spanning_tree_multilevel_after_n_iterations=5,
                             num_parts=2)
    assert e.value.rc == 5   # B2TEX_ERR_UNSUPPORTED
    info, trace = c.view_selection_run()   # the context stays usable
    assert info.iterations == r["mrf"]["iterations"] and np.array_equal(c.labels_download(), r["mrf"]["labels"])
    assert np.array_equal(trace, r["mrf"]["trace"])
    c.close()
