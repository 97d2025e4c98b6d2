"""Builds libb2tex.so (sm_90a only) in-tree with nvcc.  Used by __graft_entry__.build()."""
from __future__ import annotations

import concurrent.futures as cf
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libb2tex.so")
SOURCES = ["api.cu", "imgprep.cu", "bvh.cu", "datacosts.cu", "mrf.cu", "seam.cu", "patches.cu", "localseam.cu", "seam_mg.cu",
           "undistort.cu", "graph.cu", "prepare.cu", "mrf_multilevel.cu"]
# -fmad=false: results must match the fp32 operation order of the reference restatement (oracle/)
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-fmad=false", "-Xcompiler", "-fPIC", "-Xcompiler", "-O3", "-Xptxas", "-v",
              "-ccbin", "/usr/bin/g++"]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(HERE, "..", "include", "b2tex.h"))
    hdrs.append(os.path.abspath(__file__))   # a change of the flags rebuilds every object
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    jobs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(objdir, s.replace(".cu", ".o"))
        if force or _stale(obj, [src] + hdrs):
            jobs.append((src, obj))

    def run(job):
        src, obj = job
        r = subprocess.run([nvcc, *NVCC_FLAGS, "-c", src, "-o", obj], capture_output=True, text=True)
        return job, r

    with cf.ThreadPoolExecutor(max_workers=6) as ex:
        for (src, obj), r in ex.map(run, jobs):
            if verbose or r.returncode:
                sys.stderr.write(r.stdout + r.stderr)
            if r.returncode:
                raise RuntimeError(f"nvcc failed on {src}")
            with open(obj + ".ptxas.txt", "w") as f:
                f.write(r.stderr)
    objs = [os.path.join(objdir, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or _stale(OUT, objs):
        subprocess.check_call([nvcc, "-shared", "-o", OUT + ".tmp", *objs, "-ccbin", "/usr/bin/g++",
                               "-gencode", "arch=compute_90a,code=sm_90a"])
        os.replace(OUT + ".tmp", OUT)   # atomic: a snapshot of the tree never sees a half-written library
        import hashlib
        import time
        h = hashlib.sha256()
        for f in sorted(os.listdir(CSRC)):
            h.update(open(os.path.join(CSRC, f), "rb").read())
        with open(os.path.join(objdir, "STAMP"), "w") as f:
            f.write(f"{time.strftime('%Y-%m-%d %H:%M:%S')} csrc {h.hexdigest()[:12]}\n")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
