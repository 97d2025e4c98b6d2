"""Mesh graph on the device (b2tex_build_mesh_graph, csrc/graph.cu) against the numpy builders scene.face_adjacency /
scene.vertex_rings, on C3 (2 M faces) and on C5's mesh (10 M faces).  Prints one JSON line per mesh and a final one with
the card:

  device_ms        b2tex_build_mesh_graph, host clock around the call (it ends in a device synchronise), median of
                   --reps after --warmup calls
  event_ms         the same call between two CUDA events ("graph_build"), and per kernel group (validate, edge sort,
                   adjacency count + scan, adjacency fill, vertex -> faces, vertex -> vertices) with its algorithmic
                   bytes and GB/s, medians of a second, profiled series
  host_s           the numpy builders, timed once
  identical        the six device arrays equal the host arrays byte for byte
  gpu              name, power limit and max SM clock of the card, read in the same run

Usage: python tools/graph_bench.py [--configs C3,C5] [--reps 10] [--warmup 2] [--out FILE]
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

GROUPS = ["graph_validate", "graph_edge_sort", "graph_adj_count", "graph_adj_fill", "graph_vf", "graph_vv"]


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:   # the measurement stands without it; say so
        return f"unknown ({e})"


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

    lines = []
    for name in a.configs.split(","):
        s = scene_mod.config(name, with_images=False)
        F, Vn = s.faces.shape[0], s.verts.shape[0]
        c = b2.Context(0)
        c.set_mesh(s.verts, s.faces, s.face_normals)
        for _ in range(a.warmup):
            info = c.build_mesh_graph()
        wall = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            info = c.build_mesh_graph()
            wall.append((time.perf_counter() - t0) * 1e3)
        ev = {g: [] for g in ["graph_build"] + GROUPS}
        nbytes = {}
        for _ in range(a.reps):
            c.profile(True)
            c.build_mesh_graph()
            for n, ms, by in c.profile_report():
                ev.setdefault(n, []).append(ms)
                nbytes[n] = by
            c.profile(False)
        g = c.mesh_graph_download(info)
        c.close()

        t0 = time.perf_counter()
        ap_, ai_ = scene_mod.face_adjacency(s.faces)
        t1 = time.perf_counter()
        rings = scene_mod.vertex_rings(s.faces, Vn)
        t2 = time.perf_counter()
        host = dict(adj_ptr=ap_, adj_idx=ai_, vf_ptr=rings[0], vf_idx=rings[1], vv_ptr=rings[2], vv_idx=rings[3])
        identical = {k: bool(g[k].dtype == v.dtype and g[k].tobytes() == v.tobytes()) for k, v in host.items()}

        groups = {}
        for n in GROUPS:
            ms = statistics.median(ev[n])
            groups[n] = dict(ms=ms, bytes=nbytes.get(n, 0.0), gbps=nbytes.get(n, 0.0) / ms / 1e6 if ms > 0 else None)
        res = dict(config=name, faces=F, verts=Vn, adjacency=info.num_adjacency, vertex_neighbours=info.num_vertex_neighbours,
                   max_face_degree=info.max_face_degree, non_manifold_edges=info.num_non_manifold_edges,
                   device_ms=statistics.median(wall), device_ms_all=wall,
                   event_ms=dict(graph_build=statistics.median(ev["graph_build"]),
                                 kernel_groups_sum=sum(v["ms"] for v in groups.values()), groups=groups),
                   host_s=dict(face_adjacency=t1 - t0, vertex_rings=t2 - t1),
                   identical=identical)
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
