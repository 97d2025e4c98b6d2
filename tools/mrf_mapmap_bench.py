"""texrecon's mapMAP schedule (spanning_tree_multilevel_after_n_iterations, csrc/mrf.cu) against the default, spanning-tree
and spanning + multilevel schedules, on the device.

For each scene: data costs and the face graph on the device, then b2tex_view_selection_run with four schedules -- default,
use_spanning_tree, both flags (the post-acyclic multilevel schedule), and texrecon's control (b2tex_texrecon_mrf_params:
both flags and a multilevel step after every 5 spanning iterations) -- alternating, --warmup calls each and then --reps
timed calls each.  The call time is the host clock around the call (it ends in a device synchronise).  After the timed
calls, one profiled call per schedule gives the device time of each launch group between CUDA events (b2tex_profile),
summed over the call; a multilevel step's groups are mrf_ml.* (the contraction and the projections),
mrf.k_forest_spanning / mrf.k_tree_spanning_weighted (its coarse iteration) and mrf.accept.  Prints one JSON line per
scene and a final line with the card's name, power limit and max SM clock, read in the same run.

Usage: python tools/mrf_mapmap_bench.py [--configs C3] [--reps 5] [--warmup 1] [--out FILE]
"""
import argparse
import importlib
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from mrf_multilevel_bench import gpu_info  # noqa: E402

FLAGS = ("use_spanning_tree", "use_multilevel", "spanning_tree_multilevel_after_n_iterations")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C3")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    b2 = importlib.import_module("mvs-texturing_b200")
    scene_mod = importlib.import_module("mvs-texturing_b200.scene")
    import numpy as np

    preset = b2.texrecon_mrf_params()
    schedules = {"default": {}, "spanning": dict(use_spanning_tree=1),
                 "both": dict(use_spanning_tree=1, use_multilevel=1),
                 "texrecon": {k: getattr(preset, k) for k in FLAGS}}
    lines = []
    for name in a.configs.split(","):
        s = scene_mod.config(name)
        c = b2.Context(0)
        c.set_scene(s)
        c.build_mesh_graph()
        c.data_costs_run()
        res = {k: dict(ms=[], labels=None, same=True) for k in schedules}
        for rep in range(a.warmup + a.reps):
            for key, kw in schedules.items():
                t0 = time.perf_counter()
                info, trace = c.view_selection_run(**kw)
                ms = 1e3 * (time.perf_counter() - t0)
                labels = c.labels_download()
                r = res[key]
                if r["labels"] is None:
                    r["labels"] = labels
                else:
                    r["same"] = r["same"] and bool(np.array_equal(r["labels"], labels))
                if rep >= a.warmup:
                    r["ms"].append(ms)
                r.update(iterations=int(info.iterations), spanning=int(info.spanning_tree_iterations),
                         rejected=int(info.spanning_tree_rejected), passes=int(info.multilevel_passes),
                         steps=int(info.multilevel_steps), steps_rejected=int(info.multilevel_steps_rejected),
                         coarse_nodes=int(info.coarse_nodes), global_trees=int(info.global_trees),
                         energy=float(info.energy_final), energy_initial=float(info.energy_initial),
                         monotone=bool(np.all(np.diff(trace) <= 0)))
        for key, kw in schedules.items():   # per-stage device time of one call, in a separate profiled run
            c.profile(True)
            c.view_selection_run(**kw)
            st = {}
            for n, ms, _ in c.profile_report():
                st[n] = st.get(n, 0.0) + ms
            c.profile(False)
            res[key]["stages"] = {k: round(v, 2) for k, v in sorted(st.items(), key=lambda kv: -kv[1])}
        c.close()
        out = {"scene": name, "faces": int(s.num_faces), "views": int(s.num_views)}
        for key, r in res.items():
            out[key] = {"median_ms": round(statistics.median(r["ms"]), 2), "min_ms": round(min(r["ms"]), 2),
                        "iterations": r["iterations"], "spanning_tree_iterations": r["spanning"],
                        "acyclic_iterations": r["iterations"] - r["spanning"] if r["spanning"] and not r["passes"] else None,
                        "spanning_tree_rejected": r["rejected"], "multilevel_passes": r["passes"],
                        "multilevel_steps": r["steps"], "multilevel_steps_rejected": r["steps_rejected"],
                        "coarse_nodes": r["coarse_nodes"], "global_trees": r["global_trees"],
                        "energy": round(r["energy"], 3), "energy_initial": round(r["energy_initial"], 3),
                        "trace_monotone": r["monotone"], "repeatable": r["same"], "profiled_stage_ms": r["stages"]}
        e0 = res["default"]["energy"]
        out["energy_change_percent"] = {k: round(100.0 * (res[k]["energy"] - e0) / e0, 3) for k in schedules}
        lines.append(out)
        print(json.dumps(out), flush=True)
    tail = {"gpu": gpu_info(), "reps": a.reps, "warmup": a.warmup}
    lines.append(tail)
    print(json.dumps(tail), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
