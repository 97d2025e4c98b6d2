"""Mesh preparation on the device (b2tex_prepare_mesh, csrc/prepare.cu) against the CPU oracle (oracle/prepare_mesh.c),
on C3 (2 M faces) and on C5's mesh (10 M faces), each clean and with about 1 % redundant faces injected (reversed and
rotated duplicates, degenerate subset faces, at random positions).  Prints one JSON line per mesh and a final one with the
card:

  device_ms     b2tex_prepare_mesh, host clock around the call (it ends in a device synchronise), median of --reps after
                --warmup calls; the upload of the raw arrays is included
  event_ms      the same call between two CUDA events ("prep_mesh") and per kernel group (validate, keys + sort, runs,
                subset lookups, compaction + face normals, the graph build's groups, vertex normals) with its algorithmic
                bytes and GB/s, medians of a second, profiled series
  oracle_s      the CPU oracle (ring scan, face and vertex normals) on the same arrays, timed once
  identical     kept faces, their input ids and face normals equal the oracle's byte for byte; max_vn_diff is the largest
                vertex-normal difference (acosf may differ in the last ulp)
  gpu           name, power limit and max SM clock of the card, read in the same run

Usage: python tools/prepare_bench.py [--configs C3,C5] [--reps 10] [--warmup 2] [--out FILE]
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
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]

GROUPS = ["prep_validate", "prep_sort", "prep_runs", "prep_subsets", "prep_compact", "graph_validate", "graph_edge_sort",
          "graph_adj_count", "graph_adj_fill", "graph_vf", "graph_vv", "prep_vertex_normals"]


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:   # the measurement stands without it; say so
        return f"unknown ({e})"


def inject(np, faces, frac=0.01, seed=11):
    """faces with about frac redundant faces inserted at random positions"""
    rng = np.random.RandomState(seed)
    n = int(frac * len(faces))
    src = faces[rng.choice(len(faces), n, replace=False)].astype(np.int64)
    a, b, c = src[:, 0], src[:, 1], src[:, 2]
    kind = np.arange(n) % 4
    extra = np.where(kind[:, None] == 0, np.stack([b, c, a], 1),
                     np.where(kind[:, None] == 1, np.stack([c, b, a], 1),
                              np.where(kind[:, None] == 2, np.stack([a, a, b], 1), np.stack([c, c, c], 1))))
    pos = np.sort(rng.randint(0, len(faces) + 1, n))
    return np.ascontiguousarray(np.insert(faces, pos, extra.astype(np.uint32), axis=0), np.uint32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C3,C5")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    b2 = importlib.import_module("mvs-texturing_b200")
    scene_mod = importlib.import_module("mvs-texturing_b200.scene")
    import numpy as np
    import oracle_prepare as OP

    lines = []
    for name in a.configs.split(","):
        s = scene_mod.config(name, with_images=False)
        for variant in ("clean", "redundant"):
            faces = np.ascontiguousarray(s.faces, np.uint32) if variant == "clean" else inject(np, s.faces)
            c = b2.Context(0)
            for _ in range(a.warmup):
                info = c.prepare_mesh(s.verts, faces)
            wall = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                info = c.prepare_mesh(s.verts, faces)
                wall.append((time.perf_counter() - t0) * 1e3)
            ev, nbytes = {}, {}
            for _ in range(a.reps):
                c.profile(True)
                c.prepare_mesh(s.verts, faces)
                for n, ms, by in c.profile_report():
                    ev.setdefault(n, []).append(ms)
                    nbytes[n] = by
                c.profile(False)
            d = c.prepared_mesh_download(info)
            c.close()

            t0 = time.perf_counter()
            o = OP.prepare_mesh(s.verts, faces)
            oracle_s = time.perf_counter() - t0
            identical = dict(faces=d["faces"].tobytes() == o["faces"].tobytes(), kept=d["kept"].tobytes() == o["kept"].tobytes(),
                             face_normals=d["face_normals"].tobytes() == o["face_normals"].tobytes(),
                             num_redundant=int(info.num_redundant) == o["num_redundant"])
            groups = {}
            for n in GROUPS:
                if n in ev:
                    ms = statistics.median(ev[n])
                    groups[n] = dict(ms=ms, bytes=nbytes[n], gbps=nbytes[n] / ms / 1e6 if ms > 0 else None)
            res = dict(config=name, variant=variant, faces_in=len(faces), faces=int(info.num_faces), verts=len(s.verts),
                       redundant=int(info.num_redundant), zero_normals=int(info.num_zero_normals),
                       device_ms=statistics.median(wall), device_ms_all=wall,
                       event_ms=dict(prep_mesh=statistics.median(ev["prep_mesh"]),
                                     kernel_groups_sum=sum(v["ms"] for v in groups.values()), groups=groups),
                       oracle_s=oracle_s, identical=identical,
                       max_vn_diff=float(np.abs(d["vertex_normals"] - o["vertex_normals"]).max()))
            line = json.dumps(res)
            print(line, flush=True)
            lines.append(line)
    line = json.dumps(dict(gpu=gpu_info()))
    print(line)
    lines.append(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")
    if not all(all(json.loads(l).get("identical", {}).values()) for l in lines):
        sys.exit(1)


if __name__ == "__main__":
    main()
