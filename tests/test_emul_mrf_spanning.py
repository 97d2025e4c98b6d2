"""Spanning-tree view selection's device code on the fiber emulator, against the oracle (oracle/mrf_spanning.c): one
iteration of csrc/mrf.cu's k_forest<true>, k_tree_prep<true>, k_tree<G, 3, false, true>, k_energy, k_accept and k_restore
(tests/cpp/emul_mrf_spanning.cpp) gives the oracle's levels, parents, swept labels, accept decision and final labels."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_cuda_emulation import _kernel_part
from test_mrf_spanning_cpu import _argmin_start, path_rejection_mrf, rejection_iteration

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mvs-texturing_b200", "csrc")
CPP = os.path.join(ROOT, "tests", "cpp")
OUT = os.path.join(CPP, "_emul", "spanning")
CUDA_INC = "/usr/local/cuda/include"

pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")),
                                reason="CUDA headers not installed")

SCENES = ["tiny", "occ", "messy", "C2s"]


@pytest.fixture(scope="module")
def emul():
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "mrf_kernels.inc"), "w") as f:
        f.write(_kernel_part("mrf.cu", "Mrf make_mrf(b2tex_ctx",
                             [("// ---- shared-memory / async-copy primitives", "// ---- end of primitives ----"),
                              ("// ---- system-scope flag primitives", "// ---- end of flag primitives ----")],
                             "    extern __shared__ __align__(16) unsigned char tree_dyn[];\n", close=2))
    so = os.path.join(OUT, "emul_mrf_spanning.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                           "-w", "-I" + os.path.join(CPP, "emul_include"), "-I" + CPP, "-I" + CUDA_INC, "-I" + CSRC,
                           "-I" + OUT, os.path.join(CPP, "emul_mrf_spanning.cpp"), "-o", so])
    return C.CDLL(so)


@pytest.fixture(scope="module")
def st():
    import oracle_spanning as OS
    OS.lib()
    return OS


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _check(emul, st, ap, ai, fp, view, cost, K, labels, t, group, cap, **kw):
    ap, ai = np.ascontiguousarray(ap, np.uint32), np.ascontiguousarray(ai, np.uint32)
    fp, view, cost = np.ascontiguousarray(fp, np.uint64), np.ascontiguousarray(view, np.uint16), np.ascontiguousarray(cost, np.float32)
    o = st.spanning_iteration(ap, ai, fp, view, cost, labels, t, **kw)
    import oracle as O
    pr = O.mrf_params(**kw)
    F = len(fp) - 1
    got = np.array(labels, np.uint32)
    level, parent, swept = np.zeros(F, np.uint32), np.zeros(F, np.uint32), np.zeros(F, np.uint32)
    rej, slow = C.c_uint32(), C.c_ulonglong()
    params = np.array([pr.root_div, pr.seed, t, group, cap], np.uint32)
    rc = emul.emul_spanning_iteration(C.c_uint32(F), C.c_uint32(K), _p(ap), _p(ai), _p(fp), _p(view), _p(cost), _p(params),
                                      _p(got), _p(level), _p(parent), _p(swept), C.byref(rej), C.byref(slow))
    assert rc == 0
    assert np.array_equal(level, o["level"]), (t, group, cap)
    assert np.array_equal(parent, o["parent"]), (t, group, cap)
    assert np.array_equal(swept, o["swept"]), (t, group, cap)
    assert bool(rej.value) == o["rejected"], (t, group, cap)
    assert np.array_equal(got, o["labels"]), (t, group, cap)
    return o, slow.value


@pytest.mark.parametrize("name", SCENES)
def test_spanning_iteration_matches_oracle(emul, st, oracle_pipeline, get_scene, name):
    """the first two iterations of the spanning phase, for lane groups of 4 and 32, and with a 16-label scratch that sends
    long lists through the global-memory recursion"""
    r = oracle_pipeline(name, ("dc", "mrf"))
    dc = r["dc"]
    ap, ai = r["adj"]
    K = get_scene(name).num_views
    labels = _argmin_start(dc["face_ptr"], dc["view"], dc["cost"])
    slow = 0
    for t in (1, 2):
        for group, cap in ((4, 0), (32, 0), (8, 16)):
            o, s = _check(emul, st, ap, ai, dc["face_ptr"], dc["view"], dc["cost"], K, labels, t, group, cap)
            slow += s
        labels = o["labels"]
    if name == "messy":   # non-manifold fins: trees with a node of degree > 3 take the global-memory recursion
        assert slow > 0


def test_rejected_iteration_matches_oracle(emul, st):
    ap, ai, fp, view, cost = path_rejection_mrf()
    t = rejection_iteration(st)
    start = np.array([1, 1, 2, 2], np.uint32)
    for group, cap in ((4, 0), (32, 0)):
        o, _ = _check(emul, st, ap, ai, fp, view, cost, 2, start, t, group, cap)
        assert o["rejected"] and np.array_equal(o["labels"], start)
