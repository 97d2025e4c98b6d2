"""Multilevel view selection (use_multilevel, csrc/mrf_multilevel.cu) against the default schedule, on the device.

For each scene: data costs and the face graph on the device, then b2tex_view_selection_run with use_multilevel = 0 and 1,
alternating, --warmup calls each and then --reps timed calls each.  The call time is the host clock around the call, not a
pair of CUDA events: the call reads the stop flag and the contraction's sizes back on the host between its launches, and it
ends in a device synchronise, so the host clock is the time a caller waits.  After the timed calls, one profiled call per
schedule gives the device time of each launch group between CUDA events (b2tex_profile), summed over the call: the forest
sampling, the tree DP (unweighted on the faces, weighted on the contracted MRF), the energy, and the multilevel stages
(mrf_ml.contract with its parts components / numbering / label_lists / edges, and mrf_ml.project).  Prints one JSON line per
scene (median and min milliseconds, per-stage milliseconds, iterations, energies, passes, coarse nodes, whether repeated runs
gave the same labels) and a final line with the card's name, power limit and max SM clock, read in the same run.

Usage: python tools/mrf_multilevel_bench.py [--configs C3] [--reps 5] [--warmup 1] [--out FILE]
"""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:   # the measurement stands without it; say so
        return f"unknown ({e})"


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

    lines = []
    for name in a.configs.split(","):
        s = scene_mod.config(name)
        c = b2.Context(0)
        c.set_scene(s)
        c.build_mesh_graph()
        c.data_costs_run()
        res = {}
        for flag in (0, 1):
            res[flag] = dict(ms=[], labels=None, same=True)
        for rep in range(a.warmup + a.reps):
            for flag in (0, 1):
                t0 = time.perf_counter()
                info, trace = c.view_selection_run(use_multilevel=flag)
                ms = 1e3 * (time.perf_counter() - t0)
                labels = c.labels_download()
                r = res[flag]
                if r["labels"] is None:
                    r["labels"] = labels
                else:
                    r["same"] = r["same"] and bool(np.array_equal(r["labels"], labels))
                if rep >= a.warmup:
                    r["ms"].append(ms)
                r.update(iterations=int(info.iterations), energy=float(info.energy_final),
                         energy_initial=float(info.energy_initial), passes=int(info.multilevel_passes),
                         coarse_nodes=int(info.coarse_nodes), monotone=bool(np.all(np.diff(trace) <= 0)))
        for flag in (0, 1):   # per-stage device time of one call, in a separate profiled run
            c.profile(True)
            c.view_selection_run(use_multilevel=flag)
            st = {}
            for n, ms, _ in c.profile_report():
                st[n] = st.get(n, 0.0) + ms
            c.profile(False)
            res[flag]["stages"] = {k: round(v, 2) for k, v in sorted(st.items(), key=lambda kv: -kv[1])}
        c.close()
        out = {"scene": name, "faces": int(s.num_faces), "views": int(s.num_views)}
        for flag, key in ((0, "default"), (1, "multilevel")):
            r = res[flag]
            out[key] = {"median_ms": round(statistics.median(r["ms"]), 2), "min_ms": round(min(r["ms"]), 2),
                        "iterations": r["iterations"], "energy": round(r["energy"], 3),
                        "energy_initial": round(r["energy_initial"], 3), "multilevel_passes": r["passes"],
                        "coarse_nodes": r["coarse_nodes"], "trace_monotone": r["monotone"],
                        "repeatable": r["same"], "profiled_stage_ms": r["stages"]}
        e0, e1 = res[0]["energy"], res[1]["energy"]
        out["energy_change_percent"] = round(100.0 * (e1 - e0) / e0, 3)
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
