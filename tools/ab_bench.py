#!/usr/bin/env python
"""A/B timing of two trees of this project on one GPU: runs each tree's own bench.py in alternation, N times each.

    python tools/ab_bench.py --base /path/to/baseline_tree [--new .] --runs 3 [--steps 5 --warmup 3 --workload C3]
                             [--out DIR]

Both trees must have been built (libb2tex.so next to their package).  Per run it prints ms_per_step,
stage_ms.data_costs and .seam_leveling, the k_pcg time (its own events), the data-cost kernel groups bench.py reports,
verify.crc_data_costs / crc_labels and the
verify flags; every run also writes `--dump-outputs` to DIR/<label>_<i>/, and the outputs of all runs are compared
byte for byte (by sha256; the dumps are removed afterwards unless --keep-dumps).  Then one profiling pass per tree
(same workload, profiler on) lists EVERY kernel group of the data-cost stage, including those below bench.py's top ten.  The GPU name and power limit are read in the same invocation.
Spread = max - min of a build's ms_per_step; the gain is judged against it.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile

DC_PREFIXES = ("k_cull", "k_rays", "k_quality", "k_outlier", "k_count_survivors", "k_compact", "k_histogram",
               "k_normalize", "bvh", "k_morton", "k_hierarchy", "k_refit", "k_lum", "k_sobel")

PROFILE = r"""
import importlib, json, sys
import torch
tree, workload, steps, warmup = sys.argv[1], sys.argv[2], int(sys.argv[3]), int(sys.argv[4])
sys.path.insert(0, tree)
import bench
b2 = importlib.import_module("mvs-texturing_b200")
scene_mod = importlib.import_module("mvs-texturing_b200.scene")
par = importlib.import_module("mvs-texturing_b200.sharded")
s, adj, rings, _ = bench.build_workload(scene_mod, workload)
runner = par.ShardedPipeline(b2, s, adj, rings, 0, 1, 0)
for _ in range(warmup):
    runner.step()
torch.cuda.synchronize()
runner.ctx.profile(True)
for _ in range(steps):
    runner.step()
torch.cuda.synchronize()
agg = {}
for name, ms, by in runner.ctx.profile_report():
    a = agg.setdefault(name, [0, 0.0, 0.0])
    a[0] += 1; a[1] += ms; a[2] += by
runner.ctx.profile(False)
print(json.dumps({n: {"launch_groups": c / steps, "ms_per_step": ms / steps, "gbs": by / ms / 1e6 if ms else 0.0}
                  for n, (c, ms, by) in agg.items()}), flush=True)
"""


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi failed)"
    except (OSError, subprocess.SubprocessError):
        return "unknown (nvidia-smi unavailable)"


def last_json(text):
    for line in reversed(text.splitlines()):
        line = line.strip()
        if line.startswith("{"):
            return json.loads(line)
    raise RuntimeError("no JSON line in the output:\n" + text[-4000:])


def run_bench(tree, args, dump):
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(args.steps), "--warmup", str(args.warmup),
           "--workload", args.workload, "--no-cpu-baseline", "--no-e2e", "--dump-outputs", dump]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=tree)
    if r.returncode:
        raise RuntimeError(f"{' '.join(cmd)} failed ({r.returncode}):\n{r.stderr[-4000:]}")
    return last_json(r.stdout)


def digest(d):
    """sha256 of every file of a dump directory"""
    return {f: hashlib.sha256(open(os.path.join(d, f), "rb").read()).hexdigest() for f in sorted(os.listdir(d))}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--base", required=True, help="baseline tree (built)")
    ap.add_argument("--new", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))), help="tree under test (built)")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workload", default="C3")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "ab_bench"))
    ap.add_argument("--no-profile", action="store_true", help="skip the per-tree profiling pass")
    ap.add_argument("--keep-dumps", action="store_true", help="keep the output dumps (tens of MB per run) after hashing them")
    args = ap.parse_args()
    trees = {"base": os.path.abspath(args.base), "new": os.path.abspath(args.new)}
    os.makedirs(args.out, exist_ok=True)
    gpu = gpu_info()
    print(f"GPU (name, power limit, max SM clock): {gpu}", flush=True)
    rows = {k: [] for k in trees}
    for i in range(args.runs):
        order = ("base", "new") if i % 2 == 0 else ("new", "base")   # alternate which build runs first
        for label in order:
            dump = os.path.abspath(os.path.join(args.out, f"{label}_{i}"))
            res = run_bench(trees[label], args, dump)
            with open(os.path.join(args.out, f"{label}_{i}.json"), "w") as f:
                json.dump(res, f)
            v = res.get("verify") or {}
            kern = {k["name"]: round(k["ms_per_step"], 3) for k in res["kernels"] if k["name"].startswith(DC_PREFIXES)}
            pcg = next((k for k in res["kernels"] if k["name"] in ("k_pcg", "k_pcg_mg")), None)
            row = {"build": label, "run": i, "ms_per_step": round(res["ms_per_step"], 2),
                   "data_costs_ms": round(res["stage_ms"].get("data_costs", float("nan")), 2), "dc_kernels_top10": kern,
                   "seam_leveling_ms": round(res["stage_ms"].get("seam_leveling", float("nan")), 2),
                   "k_pcg_ms": round(pcg["ms_per_step"], 3) if pcg else None,
                   "verify_ok": v.get("ok"), "data_costs_bit_exact": v.get("data_costs_bit_exact"),
                   "labels_bit_exact": v.get("labels_bit_exact"), "mrf_energy_identical": v.get("mrf_energy_identical"),
                   "crc_data_costs": v.get("crc_data_costs"), "crc_labels": v.get("crc_labels"),
                   "clocks": res.get("clocks"), "dump_sha256": digest(dump)}
            if not args.keep_dumps:
                shutil.rmtree(dump)
            rows[label].append(row)
            print(json.dumps(row), flush=True)

    summary = {"gpu": gpu, "workload": args.workload, "steps": args.steps, "warmup": args.warmup}
    for label, rs in rows.items():
        ms = [r["ms_per_step"] for r in rs]
        dc = [r["data_costs_ms"] for r in rs]
        sl = [r["seam_leveling_ms"] for r in rs]
        pcg = [r["k_pcg_ms"] for r in rs if r["k_pcg_ms"] is not None]
        summary[label] = {"ms_per_step": ms, "median": sorted(ms)[len(ms) // 2], "spread": max(ms) - min(ms),
                          "data_costs_ms": dc, "data_costs_median": sorted(dc)[len(dc) // 2],
                          "seam_leveling_ms": sl, "k_pcg_ms": pcg, "k_pcg_median": sorted(pcg)[len(pcg) // 2] if pcg else None}
    summary["gain_ms"] = summary["base"]["median"] - summary["new"]["median"]
    summary["gain_over_3x_spread"] = summary["gain_ms"] > 3 * max(summary["base"]["spread"], summary["new"]["spread"])
    all_rows = rows["base"] + rows["new"]
    summary["crc_identical"] = (len({json.dumps(r["crc_data_costs"]) for r in all_rows}) == 1
                                and len({r["crc_labels"] for r in all_rows}) == 1)
    summary["verify_all"] = all(r["verify_ok"] and r["data_costs_bit_exact"] and r["labels_bit_exact"] and r["mrf_energy_identical"]
                                for r in all_rows)
    summary["dumps_identical"] = all(r["dump_sha256"] == all_rows[0]["dump_sha256"] for r in all_rows[1:])

    if not args.no_profile:
        for label, tree in trees.items():
            r = subprocess.run([sys.executable, "-c", PROFILE, tree, args.workload, str(args.steps), str(args.warmup)],
                               capture_output=True, text=True, cwd=tree)
            if r.returncode:
                summary[f"profile_{label}"] = f"failed: {r.stderr[-2000:]}"
                continue
            groups = last_json(r.stdout)
            summary[f"profile_{label}"] = {n: {"ms": round(g["ms_per_step"], 3), "gbs": round(g["gbs"], 1)}
                                           for n, g in sorted(groups.items(), key=lambda kv: -kv[1]["ms_per_step"])
                                           if n.startswith(DC_PREFIXES)}
    print(json.dumps(summary, indent=1), flush=True)
    with open(os.path.join(args.out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
