"""Solver quality study (CPU, oracle): energy of the forest block-coordinate-descent solver at its stop rule, after 200
iterations, and with the spanning-tree, multilevel and texrecon (mapMAP's control in view_selection.cpp:103-115) schedules, against two lower bounds of the optimum of the SAME model (view_selection.cpp:26-90: unaries = data costs, unit
Potts edges between seen adjacent faces, unseen faces cost 1):
  LB_unary : sum of the cheapest label of every face (all pairwise terms >= 0)
  LB_tree  : exact optimum (min-sum DP) of the model with only the edges of a BFS spanning forest kept -- dropping
             non-negative terms can only lower the minimum, so it bounds the optimum of the full model from below.
mapMAP itself is absent (DESIGN.md section 2), so this is the yardstick for "how far from optimal can the labeling be".

    python tools/mrf_quality.py C1 C1d C2s C3s          # writes profiles/r02_mrf_quality.md
"""
import importlib, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "oracle"))
import oracle as O
import oracle_multilevel as OM
import oracle_spanning as OS
import oracle_mapmap as OMM
scene = importlib.import_module("mvs-texturing_b200.scene")


def tree_lower_bound(ap, ai, fp, view, cost):
    F = len(fp) - 1
    n = np.diff(fp).astype(np.int64)
    seen = n > 0
    parent = np.full(F, -1, np.int64)
    order = []
    visited = ~seen            # unseen faces carry no edges: constant cost 1 each
    for root in range(F):
        if visited[root]:
            continue
        visited[root] = True
        q = [root]
        while q:
            nq = []
            for v in q:
                order.append(v)
                for w in ai[ap[v]:ap[v + 1]]:
                    if not visited[w]:
                        visited[w] = True; parent[w] = v; nq.append(w)
            q = nq
    h = [None] * F
    total = float((~seen).sum())
    for v in order:
        h[v] = cost[fp[v]:fp[v + 1]].astype(np.float64).copy()
    for v in reversed(order):   # children before parents (BFS order reversed)
        p = parent[v]
        hv = h[v]
        hmin = hv.min()
        if p < 0:
            total += hmin
            continue
        lv, lp = view[fp[v]:fp[v + 1]], view[fp[p]:fp[p + 1]]
        msg = np.full(len(lp), hmin + 1.0)
        idx = np.searchsorted(lv, lp)
        ok = (idx < len(lv))
        ok[ok] &= lv[idx[ok]] == lp[ok]
        msg[ok] = np.minimum(hv[idx[ok]], hmin + 1.0)
        h[p] = h[p] + msg
    # top-down: the labeling that attains the bound (what a spanning-tree step of the solver would propose)
    labels = np.zeros(F, np.uint32)
    for v in order:
        p = parent[v]
        hv, lv = h[v], view[fp[v]:fp[v + 1]]
        k = int(np.argmin(hv))
        if p >= 0:
            want = labels[p] - 1
            j = int(np.searchsorted(lv, want))
            if j < len(lv) and lv[j] == want and hv[j] <= hv.min() + 1.0:
                k = j
        labels[v] = int(lv[k]) + 1
    return total, labels


def main(names):
    rows = []
    for name in names:
        s = scene.config(name)
        ap, ai = scene.face_adjacency(s.faces)
        o = O.data_costs(s)
        fp, view, cost = o["face_ptr"], o["view"], o["cost"]
        t0 = time.time()
        m = O.view_selection(ap, ai, fp, view, cost)
        t1 = time.time()
        m200 = O.view_selection(ap, ai, fp, view, cost, max_iterations=200, window=10 ** 6)
        ml = OM.view_selection(ap, ai, fp, view, cost, use_multilevel=1)   # multilevel schedule, default stop rule
        sp = OS.view_selection(ap, ai, fp, view, cost)                     # spanning phase, then the acyclic one
        spml = OS.view_selection(ap, ai, fp, view, cost, use_multilevel=1)
        tr = OMM.view_selection(ap, ai, fp, view, cost, n=5)                 # texrecon: a multilevel step every 5
        n = np.diff(fp)
        lb_unary = float(sum(cost[fp[v]:fp[v + 1]].min() if n[v] else 1.0 for v in range(len(n))))
        lb_tree, tree_labels = tree_lower_bound(ap, ai, fp, view, cost)
        e_tree_labels = O.mrf_energy(ap, ai, fp, view, cost, tree_labels)   # full model, all edges
        rows.append((name, s.num_faces, m["energy_initial"], m["iterations"], m["energy"], m200["energy"], lb_unary, lb_tree, e_tree_labels,
                     ml["iterations"], ml["energy"], ml["multilevel_passes"],
                     sp["spanning_tree_iterations"], sp["acyclic_iterations"], sp["spanning_tree_rejected"], sp["energy"],
                     spml["iterations"], spml["energy"],
                     tr["spanning_tree_iterations"], tr["multilevel_steps"], tr["multilevel_steps_rejected"],
                     tr["acyclic_iterations"], tr["energy"]))
        print(rows[-1], f"({t1 - t0:.1f}s)", flush=True)
    out = ["# MRF solver quality (oracle = CUDA path bit for bit; `python tools/mrf_quality.py`)", "",
           "| scene | faces | E arg-min unaries | E of the spanning-forest optimum (all edges counted) | stop rule: iterations | E at the stop rule | E after 200 iterations | LB unaries | LB spanning forest | (E_stop - LB_tree) / LB_tree | (E_stop - E_200) / E_200 | multilevel: iterations (passes) | E multilevel | (E_ml - E_stop) / E_stop | spanning: spanning + acyclic iterations (rejected) | E spanning | (E_sp - E_stop) / E_stop | spanning + multilevel: iterations | E spanning + multilevel | (E_spml - E_stop) / E_stop | texrecon: spanning (steps, rejected) + acyclic iterations | E texrecon | (E_tr - E_stop) / E_stop |",
           "|---|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|"]
    for r in rows:
        out.append(f"| {r[0]} | {r[1]} | {r[2]:.1f} | {r[8]:.1f} | {r[3]} | {r[4]:.1f} | {r[5]:.1f} | {r[6]:.1f} | {r[7]:.1f} | {100 * (r[4] - r[7]) / r[7]:.2f} % | {100 * (r[4] - r[5]) / r[5]:.2f} % | {r[9]} ({r[11]}) | {r[10]:.1f} | {100 * (r[10] - r[4]) / r[4]:.2f} % "
                   f"| {r[12]} + {r[13]} ({r[14]}) | {r[15]:.1f} | {100 * (r[15] - r[4]) / r[4]:.2f} % | {r[16]} | {r[17]:.1f} | {100 * (r[17] - r[4]) / r[4]:.2f} % "
                   f"| {r[18]} ({r[19]}, {r[20]}) + {r[21]} | {r[22]:.1f} | {100 * (r[22] - r[4]) / r[4]:.2f} % |")
    out += ["", "LB spanning forest keeps F - 1 of the ~1.5 F edges, so the true optimum lies between it and E after 200 iterations.",
            "The second energy column is the labeling that is optimal on one BFS spanning forest of the faces (all of them rooted at",
            "the lowest face of a component), scored on the full model.",
            "The multilevel columns run the use_multilevel schedule (oracle/mrf_multilevel.c) with the default stop rule and 100 iterations at",
            "most; passes = contractions whose coarse solve lowered the energy.",
            "The spanning columns run the use_spanning_tree schedule (oracle/mrf_spanning.c): spanning-forest iterations until the stop",
            "rule fires (rejected = iterations that raised the energy and were undone), then the acyclic iterations with the window",
            "restarted, 100 iterations at most in all; the spanning + multilevel columns add the multilevel schedule after them.",
            "The texrecon columns run mapMAP's control as texrecon sets it (oracle/mrf_mapmap.c, b2tex_texrecon_mrf_params): a",
            "multilevel step (one spanning-tree iteration on the contracted MRF) after every 5 spanning iterations, counted in the",
            "spanning phase's iterations; rejected = steps that raised the energy and were undone; then the acyclic phase, and",
            "nothing after it."]
    open(os.path.join(ROOT, "profiles", "r02_mrf_quality.md"), "w").write("\n".join(out) + "\n")


if __name__ == "__main__":
    main(sys.argv[1:] or ["C1", "C1d", "C2s", "C3s"])
