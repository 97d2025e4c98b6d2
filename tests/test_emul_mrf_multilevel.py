"""Multilevel view selection's device code on the host emulators, against the oracle (oracle/mrf_multilevel.c):
  * the contraction kernels of csrc/mrf_multilevel.cu (tests/cpp/emul_mrf_contract.cpp, serial emulator, CUB sorts and
    scans replaced by stable host sorts and scans): node of every face, coarse labels and label positions, label lists
    and cost sums, CSR and weights, byte for byte;
  * one iteration of csrc/mrf.cu's forest BCD with the weighted k_tree<G, 3, true> on those contracted MRFs
    (tests/cpp/emul_mrf_multilevel.cpp, fiber emulator), label for label."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_cuda_emulation import _kernel_part

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mvs-texturing_b200", "csrc")
CPP = os.path.join(ROOT, "tests", "cpp")
OUT = os.path.join(CPP, "_emul", "multilevel")
CUDA_INC = "/usr/local/cuda/include"

pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")),
                                reason="CUDA headers not installed")

SCENES = ["tiny", "occ", "messy", "C2s"]


@pytest.fixture(scope="module")
def libs():
    os.makedirs(OUT, exist_ok=True)
    src = open(os.path.join(CSRC, "mrf_multilevel.cu")).read()
    with open(os.path.join(OUT, "mrf_multilevel_kernels.inc"), "w") as f:
        f.write(src.split("template <typename T>\nint exclusive_sum")[0].replace("#include <cub/cub.cuh>", "")
                + "}  // namespace\n}  // namespace b2\n")
    with open(os.path.join(OUT, "mrf_kernels.inc"), "w") as f:
        f.write(_kernel_part("mrf.cu", "Mrf make_mrf(b2tex_ctx",
                             [("// ---- shared-memory / async-copy primitives", "// ---- end of primitives ----"),
                              ("// ---- system-scope flag primitives", "// ---- end of flag primitives ----")],
                             "    extern __shared__ __align__(16) unsigned char tree_dyn[];\n", close=2))
    out = {}
    for name, extra in (("emul_mrf_contract", []), ("emul_mrf_multilevel", ["-I" + os.path.join(CPP, "emul_include")])):
        so = os.path.join(OUT, name + ".so")
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                               "-w", *extra, "-I" + CPP, "-I" + CUDA_INC, "-I" + CSRC, "-I" + OUT,
                               os.path.join(CPP, name + ".cpp"), "-o", so])
        out[name] = C.CDLL(so)
    return out


@pytest.fixture(scope="module")
def ml():
    import oracle_multilevel as OM
    OM.lib()
    return OM


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _labelings(ml, r):
    """the labels the schedule contracts first, and a random one with large regions"""
    dc = r["dc"]
    ap, ai = r["adj"]
    first = ml.view_selection(ap, ai, dc["face_ptr"], dc["view"], dc["cost"], use_multilevel=1)["first_labels"]
    fp = dc["face_ptr"].astype(np.int64)
    n = np.diff(fp)
    rng = np.random.default_rng(11)
    pick = rng.integers(0, np.maximum(n, 1))
    pick[rng.random(len(n)) < 0.8] = 0
    rand = np.where(n > 0, dc["view"][np.minimum(fp[:-1] + pick, max(len(dc["view"]) - 1, 0))].astype(np.uint32) + 1, 0)
    return [first, rand.astype(np.uint32)]


def _check_contraction(libs, ml, ap, ai, dc, labels):
    """emulated contraction kernels == orc_mrf_contract, and no kernel writes past the device's scratch sizes"""
    o = ml.contract(ap, ai, dc["face_ptr"], dc["view"], dc["cost"], labels)
    F, nnz, A = len(labels), len(dc["view"]), len(ai)
    g = dict(region=np.zeros(F, np.uint32), labels=np.zeros(F, np.uint32), lidx=np.zeros(F, np.uint32),
             ptr=np.zeros(F + 1, np.uint64), view=np.zeros(nnz + 1, np.uint16), cost=np.zeros(nnz + 1, np.float32),
             adj_ptr=np.zeros(F + 1, np.uint32), adj_idx=np.zeros(A + 1, np.uint32), weight=np.zeros(A + 1, np.float32))
    n, rounds = C.c_uint32(), C.c_uint32()
    rc = libs["emul_mrf_contract"].emul_contract(
        C.c_uint32(F), _p(ap), _p(ai), _p(dc["face_ptr"]), _p(dc["view"]), _p(dc["cost"]), _p(labels), 3, 64,
        C.byref(n), *[_p(g[k]) for k in ("region", "labels", "lidx", "ptr", "view", "cost", "adj_ptr", "adj_idx", "weight")],
        C.byref(rounds))
    assert rc == 0
    n = n.value
    assert n == o["num_nodes"]
    nz, ne = int(o["ptr"][-1]), int(o["adj_ptr"][-1])
    assert np.array_equal(g["region"], o["region"])
    assert np.array_equal(g["labels"][:n], o["labels"])
    assert np.array_equal(g["ptr"][:n + 1], o["ptr"])
    assert np.array_equal(g["view"][:nz], o["view"])
    assert np.array_equal(g["cost"][:nz].view(np.uint32), o["cost"].view(np.uint32))
    assert np.array_equal(g["adj_ptr"][:n + 1], o["adj_ptr"])
    assert np.array_equal(g["adj_idx"][:ne], o["adj_idx"])
    assert np.array_equal(g["weight"][:ne].view(np.uint32), o["weight"].view(np.uint32))
    for v in range(n):   # the label's position in the node's list (0 for unseen nodes)
        lst = o["view"][o["ptr"][v]:o["ptr"][v + 1]].astype(np.int64) + 1
        assert g["lidx"][v] == (int(np.flatnonzero(lst == o["labels"][v])[0]) if len(lst) else 0)


@pytest.mark.parametrize("name", SCENES)
def test_contraction_kernels_match_oracle(libs, ml, oracle_pipeline, name):
    r = oracle_pipeline(name, ("dc", "mrf"))
    for labels in _labelings(ml, r):
        _check_contraction(libs, ml, *r["adj"], r["dc"], labels)


def test_contraction_of_a_triangle_soup_with_unseen_faces(libs, ml):
    """more faces than candidates and adjacency entries (no edges, 10 of 100 faces seen): the per-face phase of the
    contraction must fit the scratch"""
    F = 100
    rng = np.random.default_rng(5)
    seen = np.zeros(F, bool)
    seen[rng.choice(F, 10, replace=False)] = True
    n = np.where(seen, 2, 0)
    fp = np.concatenate([[0], np.cumsum(n)]).astype(np.uint64)
    view = np.array(sum([sorted(rng.choice(6, 2, replace=False).tolist()) for _ in range(10)], []), np.uint16)
    cost = rng.random(len(view)).astype(np.float32)
    labels = np.zeros(F, np.uint32)
    labels[seen] = view[fp[:-1][seen].astype(np.int64)].astype(np.uint32) + 1
    ap, ai = np.zeros(F + 1, np.uint32), np.zeros(0, np.uint32)
    _check_contraction(libs, ml, ap, ai, dict(face_ptr=fp, view=view, cost=cost), labels)


@pytest.mark.parametrize("name", SCENES)
def test_weighted_tree_iteration_matches_oracle(libs, ml, orc, oracle_pipeline, get_scene, name):
    """one coarse iteration (k_forest, k_tree_prep, k_tree<G, 3, true>) at the iteration numbers the schedule uses, for
    lane groups of 4 and 32, and with a 16-label scratch that sends long lists through the global-memory recursion"""
    r = oracle_pipeline(name, ("dc", "mrf"))
    dc = r["dc"]
    ap, ai = r["adj"]
    K = get_scene(name).num_views
    pr = orc.mrf_params()
    for labels in _labelings(ml, r):
        o = ml.contract(ap, ai, dc["face_ptr"], dc["view"], dc["cost"], labels)
        n = o["num_nodes"]
        for t in (9, 19, 20):
            want = o["labels"].copy()
            ml.lib().orc_mrf_sweep(C.c_uint32(n), _p(o["adj_ptr"]), _p(o["adj_idx"]), _p(o["weight"]), _p(o["ptr"]),
                                   _p(o["view"]), _p(o["cost"]), C.byref(pr), C.c_uint32(t), _p(want))
            for group, cap in ((4, 0), (32, 0), (8, 16)):
                got = o["labels"].copy()
                params = np.array([pr.rounds, pr.root_div, pr.seed, t, group, cap], np.uint32)
                slow = C.c_ulonglong()
                rc = libs["emul_mrf_multilevel"].emul_coarse_iteration(
                    C.c_uint32(n), C.c_uint32(K), _p(o["adj_ptr"]), _p(o["adj_idx"]), _p(o["weight"]), _p(o["ptr"]),
                    _p(o["view"]), _p(o["cost"]), _p(params), _p(got), C.byref(slow))
                assert rc == 0
                assert np.array_equal(got, want), (t, group, cap)
