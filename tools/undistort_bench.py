"""Undistortion and the validity flood on C3-sized views (200 views at 1920x1080) with a pincushion distortion that gives
every view black corners, so that every view gets a validity mask.  Prints one JSON line:

  k_undistort      device time of the resampling launches (CUDA events, median over --reps), its algorithmic bytes
                   (3 B gathered + 3 B written per pixel), GB/s and share of the H100 SXM data sheet's 3.35 TB/s;
                   the copy back from the scratch is reported on its own
  flood            the validity flood of prepare_images (k_flood launches plus their host polls, CUDA events) and the
                   data-cost call around it
  gpu              name and power limit of the card it ran on

The mesh is a small sphere (the C3 cameras and images, not its 1M faces): the data-cost call is then mostly
prepare_images.  Usage: python tools/undistort_bench.py [--reps 5] [--views 200] [--out FILE]
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

HBM_PEAK = 3.35e12   # H100 SXM data sheet


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:   # the measurement stands without it; say so
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--views", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    b2 = importlib.import_module("mvs-texturing_b200")
    scene_mod = importlib.import_module("mvs-texturing_b200.scene")
    import numpy as np

    s = scene_mod.sphere_scene(10, a.views, 1920, 1080, displace=0.05, name="C3-views")
    K = s.num_views
    flen = np.full(K, 0.9, np.float32)
    dist = np.tile(np.array([[0.12, 0.03]], np.float32), (K, 1))   # pincushion: black corners on every view
    px = K * s.width * s.height

    c = b2.Context(0)
    views = b2.make_views(s.pos, s.viewdir, s.proj, s.w2c, s.width, s.height, s.images)
    c.set_mesh(s.verts, s.faces, s.face_normals)
    und, back = [], []
    for rep in range(a.reps + 1):   # rep 0 warms up
        c.set_views(views, K)
        c.synchronize()
        c.profile(True)
        c.undistort_views(flen, dist)
        rows = c.profile_report()
        c.profile(False)
        if rep:
            und.append(sum(ms for n, ms, _ in rows if n == "k_undistort"))
            back.append(sum(ms for n, ms, _ in rows if n == "undistort_copy_back"))
    k_ms = statistics.median(und)
    k_bytes = 6.0 * px
    res = dict(views=K, width=s.width, height=s.height, pixels=px,
               k_undistort=dict(ms=k_ms, ms_all=und, bytes=k_bytes, gbps=k_bytes / k_ms / 1e6,
                                share_of_3_35_tbps=k_bytes / (k_ms * 1e-3) / HBM_PEAK),
               copy_back=dict(ms=statistics.median(back), bytes=6.0 * px, gbps=6.0 * px / statistics.median(back) / 1e6))

    # the undistorted images stay resident: every data-cost call redoes prepare_images with all K views flagged
    flood, call = [], []
    for rep in range(a.reps + 1):
        c.synchronize()
        c.profile(True)
        t0 = time.perf_counter()
        c.data_costs_run()
        c.synchronize()
        t1 = time.perf_counter()
        rows = c.profile_report()
        c.profile(False)
        if rep:
            flood.append(sum(ms for n, ms, _ in rows if n == "k_flood"))
            call.append((t1 - t0) * 1e3)
    res["flood"] = dict(flood_ms=statistics.median(flood), flood_ms_all=flood, data_costs_call_ms=statistics.median(call))
    res["gpu"] = gpu_info()
    c.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
