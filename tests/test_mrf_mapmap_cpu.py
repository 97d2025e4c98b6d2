"""texrecon's mapMAP schedule on the CPU oracle (oracle/mrf_mapmap.c): a multilevel step after every n-th spanning
iteration, then the acyclic phase.  n = 0 is the existing schedule, steps come where they should, the trace never rises,
the coarse spanning iteration is exact on small weighted MRFs, coarse and fine energies agree after every step, a
hand-built MRF takes the rejection branch, and the preset is the control texrecon records."""
import itertools
import os

import numpy as np
import pytest

from test_mrf_spanning_cpu import _argmin_start

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCENES = ["tiny", "C1", "C1d", "C2s", "C3s", "occ", "messy"]


@pytest.fixture(scope="module")
def mm():
    import oracle_mapmap as OM
    OM.lib()
    return OM


def step_rejection_mrf():
    """a path of seven faces, labels {1, 2} everywhere, costs on a 1/8 grid (found by searching random paths): with n = 1
    the multilevel step of iteration 4 cuts the path into coarse trees whose fixed neighbours pull both sides across the
    cut, so the projected energy rises and the step is rejected"""
    ap = np.array([0, 1, 3, 5, 7, 9, 11, 12], np.uint32)
    ai = np.array([1, 0, 2, 1, 3, 2, 4, 3, 5, 4, 6, 5], np.uint32)
    fp = np.arange(0, 15, 2, dtype=np.uint64)
    view = np.array([0, 1] * 7, np.uint16)
    cost = (np.array([0, 2, 2, 4, 1, 4, 4, 0, 1, 3, 4, 0, 4, 0]) / 8.0).astype(np.float32)
    return ap, ai, fp, view, cost


def _args(r):
    dc = r["dc"]
    ap, ai = r["adj"]
    return ap, ai, dc["face_ptr"], dc["view"], dc["cost"]


def _step_iterations(run, n):
    """iteration numbers of the multilevel steps the schedule should have taken"""
    k = 0
    steps = []
    t = 0
    while t < run["spanning_tree_iterations"]:
        t += 1
        k += 1
        if k % n == 0 and t < run["spanning_tree_iterations"]:
            t += 1
            steps.append(t)
    return steps


@pytest.mark.parametrize("name", SCENES)
def test_schedule(orc, mm, oracle_pipeline, name):
    import oracle_spanning as OS
    args = _args(oracle_pipeline(name, ("dc", "mrf")))
    # n = 0: exactly orc_view_selection_st with both flags
    same = mm.view_selection(*args, n=0)
    st = OS.view_selection(*args, use_spanning_tree=1, use_multilevel=1)
    for k in ("iterations", "spanning_tree_iterations", "spanning_tree_rejected", "acyclic_iterations",
              "multilevel_passes", "coarse_nodes"):
        assert same[k] == st[k], k
    assert np.array_equal(same["labels"], st["labels"]) and np.array_equal(same["trace"], st["trace"])
    assert same["multilevel_steps"] == 0
    for n in (5, 1, 3):
        run = mm.view_selection(*args, n=n)
        assert np.all(np.diff(run["trace"]) <= 0), n
        assert run["identity_failures"] == 0
        assert run["iterations"] == run["spanning_tree_iterations"] + run["acyclic_iterations"]
        assert run["multilevel_passes"] == 0
        assert run["trace"][-1] == orc.mrf_energy_fixed(*args, run["labels"]) / 2.0 ** 32
        # steps only after spanning counts n, 2n, ...: replay the phase and compare every iteration's energy
        steps = _step_iterations(run, n)
        assert run["multilevel_steps"] == len(steps)
        labels = _argmin_start(args[2], args[3], args[4])
        for t in range(1, run["spanning_tree_iterations"] + 1):
            if t in steps:
                o = mm.step(*args, labels, t)
                assert o["coarse_energy_after"] == o["energy_after"]
                if o["rejected"]:
                    assert np.array_equal(o["labels"], labels)
            else:
                o = OS.spanning_iteration(*args, labels, t)
            labels = o["labels"]
            assert orc.mrf_energy_fixed(*args, labels) / 2.0 ** 32 == run["trace"][t], (n, t)
        # the acyclic phase runs at least `window` iterations unless the budget runs out (min_acyclic_iterations = 5)
        assert run["acyclic_iterations"] >= min(5, 100 - run["spanning_tree_iterations"])


def test_arguments(mm):
    ap, ai, fp, view, cost = step_rejection_mrf()
    for flags in ((0, 1), (1, 0), (0, 0)):
        with pytest.raises(ValueError):
            mm.view_selection(ap, ai, fp, view, cost, n=5, use_spanning_tree=flags[0], use_multilevel=flags[1])


def test_rejected_step(orc, mm):
    ap, ai, fp, view, cost = step_rejection_mrf()
    run = mm.view_selection(ap, ai, fp, view, cost, n=1, max_iterations=12)
    assert run["multilevel_steps_rejected"] >= 1
    assert np.all(np.diff(run["trace"]) <= 0)
    # replay up to the rejected step: it restores the labels from its start by projecting the old coarse labels
    labels = _argmin_start(fp, view, cost)
    import oracle_spanning as OS
    seen_rejection = False
    for t in range(1, run["spanning_tree_iterations"] + 1):
        if t % 2 == 0:
            o = mm.step(ap, ai, fp, view, cost, labels, t)
            if o["rejected"]:
                seen_rejection = True
                assert o["energy_swept"] > o["energy_before"] == o["energy_after"]
                assert np.array_equal(o["labels"], labels)
                assert not np.array_equal(o["projected"], labels)
                assert np.array_equal(o["clabels"][o["region"]], labels)
        else:
            o = OS.spanning_iteration(ap, ai, fp, view, cost, labels, t)
        labels = o["labels"]
    assert seen_rejection


def _random_graph(rng, n, K, maxl, extra):
    edges = {(int(rng.integers(0, v)), v) for v in range(1, n)}
    for _ in range(extra):
        a, b = sorted(rng.choice(n, 2, replace=False).tolist())
        edges.add((a, b))
    nb = [[] for _ in range(n)]
    for a, b in edges:
        nb[a].append(b); nb[b].append(a)
    nb = [sorted(x) for x in nb]
    ap = np.concatenate([[0], np.cumsum([len(x) for x in nb])]).astype(np.uint32)
    ai = np.array(sum(nb, []), np.uint32)
    wt = {}
    for a, b in edges:
        wt[(a, b)] = wt[(b, a)] = float(rng.integers(1, 6))
    w = np.array([wt[(v, u)] for v in range(n) for u in nb[v]], np.float32)
    lists = [sorted(rng.choice(K, int(rng.integers(1, maxl + 1)), replace=False).tolist()) for _ in range(n)]
    fp = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.uint64)
    cost = (rng.random(sum(map(len, lists))) * 4).astype(np.float32)
    return ap, ai, w, fp, np.array(sum(lists, []), np.uint16), cost, lists


def _weighted_energy(ap, ai, w, fp, view, cost, labels):
    e = 0.0
    for v in range(len(fp) - 1):
        row = view[fp[v]:fp[v + 1]].tolist()
        e += float(cost[fp[v] + row.index(labels[v] - 1)])
        for a in range(ap[v], ap[v + 1]):
            u = ai[a]
            if u > v and labels[u] != labels[v]:
                e += float(w[a])
    return e


def test_weighted_spanning_iteration_is_exact(mm):
    """on a weighted tree with one root the coarse spanning iteration reaches the exhaustive minimum; with cycles, the
    DP is exact given the fixed non-tree neighbours (exhaustive search over the labels of the forest's nodes)"""
    rng = np.random.default_rng(23)
    for case in range(60):
        n = int(rng.integers(2, 8))
        extra = 0 if case < 30 else int(rng.integers(1, 4))
        ap, ai, w, fp, view, cost, lists = _random_graph(rng, n, 4, 3, extra)
        start = _argmin_start(fp, view, cost)
        out, level, parent = mm.spanning_sweep(ap, ai, fp, view, cost, start, 1 + case, weight=w, root_div=0)
        assert np.all(level < n)   # one root: every node is in the tree
        tree = {(int(v), int(parent[v])) for v in range(n) if parent[v] != 0xFFFFFFFF}
        tree |= {(b, a) for a, b in tree}

        def cond_energy(lab):   # the DP's objective: unaries + tree edges + non-tree edges against the start labels
            e = 0.0
            for v in range(n):
                e += float(cost[fp[v] + lists[v].index(lab[v] - 1)])
                for a in range(ap[v], ap[v + 1]):
                    u = int(ai[a])
                    if (v, u) in tree:
                        e += float(w[a]) if (u > v and lab[u] != lab[v]) else 0.0
                    else:
                        e += float(w[a]) if lab[v] != start[u] else 0.0
            return e
        best = min(cond_energy([x + 1 for x in combo]) for combo in itertools.product(*lists))
        assert abs(cond_energy(out) - best) <= 1e-4, case
        if extra == 0:
            brute = min(_weighted_energy(ap, ai, w, fp, view, cost, [x + 1 for x in combo])
                        for combo in itertools.product(*lists))
            assert abs(_weighted_energy(ap, ai, w, fp, view, cost, out) - brute) <= 1e-4, case


def test_unit_weights_are_the_spanning_iteration(mm, oracle_pipeline):
    """weight NULL and all-one weights give the DP of orc_mrf_spanning_iteration, label for label"""
    import oracle_spanning as OS
    args = _args(oracle_pipeline("messy", ("dc", "mrf")))
    labels = _argmin_start(args[2], args[3], args[4])
    ones = np.ones(len(args[1]), np.float32)
    for t in (1, 2, 3):
        ref = OS.spanning_iteration(*args, labels, t)
        for w in (None, ones):
            out, level, parent = mm.spanning_sweep(*args, labels, t, weight=w)
            assert np.array_equal(out, ref["swept"]) and np.array_equal(level, ref["level"])
            assert np.array_equal(parent, ref["parent"])
        labels = ref["labels"]


def test_texrecon_preset_is_the_recorded_control(b2):
    """the preset's flags and n are the mapMAP control the recording shim captured from view_selection.cpp"""
    import refpin
    g = np.load(os.path.join(ROOT, "tests", "golden", "reference_tu.npz"))
    keys = [k for k in g.files if k.startswith("mrf_model/") and k.endswith("/params")]
    assert keys
    preset, default = b2.texrecon_mrf_params(), b2.mrf_params()
    assert default.spanning_tree_multilevel_after_n_iterations == 0
    for k in keys:
        p = dict(zip(refpin.PARAM_NAMES, g[k].tolist()))
        assert preset.use_spanning_tree == int(p["use_spanning_tree"]) == 1
        assert preset.use_multilevel == int(p["use_multilevel"]) == 1
        assert preset.spanning_tree_multilevel_after_n_iterations == int(p["multilevel_after"]) == 5
        assert int(p["use_acyclic"]) == 1 and int(p["force_acyclic"]) == 1
        assert int(p["min_acyclic_iterations"]) == preset.window == 5
        assert preset.seed == int(p["seed"]) and preset.window == int(p["window"])
    # everything else is the default
    for name, _ in b2.B2MrfParams._fields_:
        if name not in ("use_spanning_tree", "use_multilevel", "spanning_tree_multilevel_after_n_iterations"):
            assert getattr(preset, name) == getattr(default, name), name
