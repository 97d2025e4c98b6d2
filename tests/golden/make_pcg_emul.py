"""Generates tests/golden/pcg_emul.npz: the iterations, residual bits and x that k_pcg (csrc/seam.cu) computes under the
fiber emulator on hand-built Laplacian-like systems.  tests/test_emul_pcg.py runs the current k_pcg on the same systems
and requires the same bits, so a rework of the solve's memory traffic cannot change a single iterate.

    python tests/golden/make_pcg_emul.py [COMMIT]

COMMIT (default a9d9cb6, the last k_pcg before the phase rework) names the seam.cu whose kernel text is run; it is
read with `git show`, so this needs a git checkout.  The commit is stored in the file.
"""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
CSRC = os.path.join(ROOT, "mvs-texturing_b200", "csrc")
CPP = os.path.join(ROOT, "tests", "cpp")
CUDA_INC = "/usr/local/cuda/include"
GOLDEN = os.path.join(ROOT, "tests", "golden", "pcg_emul.npz")
LAM2 = np.float32(0.1) * np.float32(0.1)


def kernel_part(src):
    """seam.cu up to its host entry point, as tests/test_cuda_emulation.py cuts it"""
    return src.split("int seam_run(b2tex_ctx")[0] + "}  // namespace\n"


def build(src, out_dir, extra_flags=()):
    """compile tests/cpp/emul_pcg.cpp against the kernel text of `src` (the contents of a seam.cu)"""
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "seam_kernels.inc"), "w") as f:
        f.write(kernel_part(src))
    so = os.path.join(out_dir, "emul_pcg.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                           *extra_flags, "-I" + os.path.join(CPP, "emul_include"), "-I" + CPP, "-I" + CUDA_INC, "-I" + CSRC,
                           "-I" + out_dir, os.path.join(CPP, "emul_pcg.cpp"), "-o", so])
    return C.CDLL(so)


def make_system(R, seed, hub_len=45, zero_rhs_channel=None):
    """Symmetric graph Laplacian with both weight classes (-1, -lambda^2) plus a diagonal shift on some rows (SPD),
    some rows with only a diagonal (half of them zero), and one hub row longer than any register batch."""
    rng = np.random.default_rng(seed)
    edges = {}
    for i in range(R):
        for _ in range(3):
            j = int(rng.integers(max(0, i - 3000), min(R, i + 3000)))
            if j != i:
                edges[(min(i, j), max(i, j))] = int(rng.random() < 0.3)     # 1: seam class (-1)
    hub = R // 3
    for j in rng.choice(R, hub_len, replace=False):
        if int(j) != hub:
            edges[(min(hub, int(j)), max(hub, int(j)))] = int(rng.random() < 0.5)
    lonely = set(int(v) for v in rng.choice(R, 12, replace=False)) - {hub}
    nbr = [[] for _ in range(R)]
    for (i, j), cls in sorted(edges.items()):
        if i in lonely or j in lonely:
            continue
        nbr[i].append((j, cls))
        nbr[j].append((i, cls))
    ptr = np.zeros(R + 1, np.uint32)
    enc, diag = [], np.zeros(R, np.float32)
    zero_diag = set(sorted(lonely)[::2])
    for i in range(R):
        d = np.float32(0.0)
        enc.append(i)
        for j, cls in nbr[i]:
            enc.append(j | (0x80000000 if cls else 0))
            d = np.float32(d + (np.float32(1.0) if cls else LAM2))
        if i in lonely:
            d = np.float32(0.0) if i in zero_diag else np.float32(1.5)
        elif rng.random() < 0.05:
            d = np.float32(d + np.float32(0.5))
        diag[i] = d
        ptr[i + 1] = len(enc)
    inv = np.where(diag != 0, np.float32(1.0) / np.where(diag != 0, diag, 1), np.float32(1.0)).astype(np.float32)
    rhs = rng.standard_normal((3, R)).astype(np.float32)
    rhs[1] *= np.linspace(0.1, 3.0, R, dtype=np.float32)           # a second spectrum: channels stop in different iterations
    rhs[:, sorted(zero_diag)] = 0.0                                # a zero row cannot reduce its residual
    if zero_rhs_channel is not None:
        rhs[zero_rhs_channel] = 0.0
    return dict(ptr=ptr, enc=np.array(enc, np.uint32), diag=diag, inv=inv, rhs=np.ascontiguousarray(rhs))


# name -> (R, seed, channel with zero rhs, max_iters).  Grid 1 -> 1024 threads, pairs of rows 2048 apart.
SYSTEMS = {
    "several_pairs_tail": (9 * 1024 + 517, 1, 2, 1000),   # > 8*1024 rows, R % 2048 != 0, zero-rhs channel
    "one_pair_tail": (1024 + 333, 2, None, 1000),
    "max_iters": (4096 + 5, 3, None, 7),
}


def run(lib, sysd, max_iters):
    R = len(sysd["diag"])
    x = np.zeros((3, R), np.float32)
    st = np.zeros(16, np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib.emul_pcg(C.c_uint32(R), p(sysd["ptr"]), p(sysd["enc"]), p(sysd["diag"]), p(sysd["inv"]), p(sysd["rhs"]),
                      C.c_uint32(max_iters), p(x), p(st))
    assert rc == 0, "emulated k_pcg hung"
    return st[:7].copy(), x


def main():
    commit = sys.argv[1] if len(sys.argv) > 1 else "a9d9cb6"
    src = subprocess.check_output(["git", "show", f"{commit}:mvs-texturing_b200/csrc/seam.cu"], cwd=ROOT, text=True)
    with tempfile.TemporaryDirectory() as d:
        lib = build(src, d)
        out = {"commit": np.array(commit)}
        for name, (R, seed, zc, mi) in SYSTEMS.items():
            st, x = run(lib, make_system(R, seed, zero_rhs_channel=zc), mi)
            out[name + "/status"] = st
            out[name + "/x"] = x
            print(name, "R", R, "iterations", st[:3], "loops", st[6])
    np.savez_compressed(GOLDEN, **out)


if __name__ == "__main__":
    main()
