"""The multilevel step of texrecon's mapMAP schedule on the fiber emulator, against the oracle (oracle/mrf_mapmap.c): on
the contraction of the labels at the step (orc_mrf_contract, which tests/test_emul_mrf_multilevel.py checks against the
device's contraction kernels), csrc/mrf.cu's k_forest<true>, k_tree_prep<true>, k_tree<G, 3, true, true>, k_energy,
k_accept, k_restore and k_step_count (tests/cpp/emul_mrf_mapmap.cpp) give the oracle's coarse forest, parents, swept
coarse labels, projected labels, accept decision and final labels, byte for byte."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_cuda_emulation import _kernel_part
from test_mrf_mapmap_cpu import step_rejection_mrf
from test_mrf_spanning_cpu import _argmin_start

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mvs-texturing_b200", "csrc")
CPP = os.path.join(ROOT, "tests", "cpp")
OUT = os.path.join(CPP, "_emul", "mapmap")
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
    so = os.path.join(OUT, "emul_mrf_mapmap.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                           "-w", "-I" + os.path.join(CPP, "emul_include"), "-I" + CPP, "-I" + CUDA_INC, "-I" + CSRC,
                           "-I" + OUT, os.path.join(CPP, "emul_mrf_mapmap.cpp"), "-o", so])
    return C.CDLL(so)


@pytest.fixture(scope="module")
def mm():
    import oracle_mapmap as OM
    OM.lib()
    return OM


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _check(emul, mm, ap, ai, fp, view, cost, K, labels, t, group, cap):
    import oracle_multilevel as OML
    ap, ai = np.ascontiguousarray(ap, np.uint32), np.ascontiguousarray(ai, np.uint32)
    fp, view, cost = np.ascontiguousarray(fp, np.uint64), np.ascontiguousarray(view, np.uint16), np.ascontiguousarray(cost, np.float32)
    o = mm.step(ap, ai, fp, view, cost, labels, t)
    c = OML.contract(ap, ai, fp, view, cost, labels)
    import oracle as O
    pr = O.mrf_params()
    F, n = len(fp) - 1, c["num_nodes"]
    assert n == o["num_nodes"] and np.array_equal(c["region"], o["region"])
    got = np.array(labels, np.uint32)
    clabels = np.array(c["labels"], np.uint32)
    level, parent, swept = np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    projected = np.zeros(F, np.uint32)
    rej, slow = C.c_uint32(), C.c_ulonglong()
    params = np.array([pr.root_div, pr.seed, t, group, cap], np.uint32)
    arr = [np.ascontiguousarray(c[k], dt) for k, dt in (("region", np.uint32), ("adj_ptr", np.uint32), ("adj_idx", np.uint32),
                                                          ("weight", np.float32), ("ptr", np.uint64), ("view", np.uint16),
                                                          ("cost", np.float32))]
    rc = emul.emul_multilevel_step(C.c_uint32(F), C.c_uint32(K), _p(ap), _p(ai), _p(fp), _p(view), _p(cost), _p(got),
                                   C.c_uint32(n), *[_p(a) for a in arr], _p(clabels), _p(params), _p(level), _p(parent),
                                   _p(swept), _p(projected), C.byref(rej), C.byref(slow))
    assert rc == 0
    assert np.array_equal(level, o["level"]), (t, group, cap)
    assert np.array_equal(parent, o["parent"]), (t, group, cap)
    assert np.array_equal(swept, o["swept"]), (t, group, cap)
    assert np.array_equal(projected, o["projected"]), (t, group, cap)
    assert bool(rej.value) == o["rejected"], (t, group, cap)
    assert np.array_equal(got, o["labels"]), (t, group, cap)
    return o, slow.value


@pytest.mark.parametrize("name", SCENES)
def test_multilevel_step_matches_oracle(emul, mm, oracle_pipeline, get_scene, name):
    """the step after the first five spanning iterations, and one from the arg-min start, for lane groups of 4 and 32,
    and with a 16-label scratch that sends long lists through the global-memory recursion"""
    import oracle_spanning as OS
    r = oracle_pipeline(name, ("dc", "mrf"))
    dc = r["dc"]
    ap, ai = r["adj"]
    args = (ap, ai, dc["face_ptr"], dc["view"], dc["cost"])
    K = get_scene(name).num_views
    start = _argmin_start(dc["face_ptr"], dc["view"], dc["cost"])
    labels = start
    for t in range(1, 6):
        labels = OS.spanning_iteration(*args, labels, t)["labels"]
    slow = 0
    for lab, t in ((labels, 6), (start, 1)):
        for group, cap in ((4, 0), (32, 0), (8, 16)):
            _, s = _check(emul, mm, *args, K, lab, t, group, cap)
            slow += s
    assert slow > 0   # contracted MRFs have nodes of degree > 3: their trees take the global-memory recursion


def test_rejected_step_matches_oracle(emul, mm):
    import oracle_spanning as OS
    ap, ai, fp, view, cost = step_rejection_mrf()
    labels = _argmin_start(fp, view, cost)
    rejected = 0
    for t in range(1, 13):   # the schedule with n = 1: spanning iterations at odd t, steps at even t
        if t % 2:
            labels = OS.spanning_iteration(ap, ai, fp, view, cost, labels, t)["labels"]
            continue
        for group, cap in ((4, 0), (32, 0)):
            o, _ = _check(emul, mm, ap, ai, fp, view, cost, 2, labels, t, group, cap)
        rejected += o["rejected"]
        labels = o["labels"]
    assert rejected >= 1
