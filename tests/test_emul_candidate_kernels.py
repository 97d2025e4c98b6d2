"""The candidate kernels of csrc/datacosts.cu (k_cull<true> and k_compact run warp per face; k_count_survivors) on the
fiber emulator (tests/cpp/emul_candidates.cpp on tests/cpp/cuda_fiber.h: all lanes of a warp alive at once), against a
numpy restatement, on inputs the scene tests do not reach: more than 1024 views (pass words beyond the first 32-word
chunk), a face range of a multi-GPU shard (faces outside it keep count 0), faces without candidates, NaN qualities
(kept, like the reference's `!= 0` test) and warps that loop over many faces."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mvs-texturing_b200", "csrc")
CPP = os.path.join(ROOT, "tests", "cpp")
OUT = os.path.join(CPP, "_emul")
CUDA_INC = "/usr/local/cuda/include"

pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")),
                                reason="CUDA headers not installed")


def _kernel_part(cu_file, host_entry, drop=None):
    """Text of a .cu file up to its first host entry point, without the CUB include and the span [drop[0], drop[1])
    (as tests/test_cuda_emulation.py cuts it)."""
    head = open(os.path.join(CSRC, cu_file)).read().split(host_entry)[0].replace("#include <cub/cub.cuh>", "")
    if drop:
        a, b = head.index(drop[0]), head.index(drop[1])
        head = head[:a] + head[b:]
    return head + "}  // namespace\n"


@pytest.fixture(scope="module")
def lib():
    inc = os.path.join(OUT, "cand")   # own directory and library name: the other emulation module may hold its build open
    os.makedirs(inc, exist_ok=True)
    with open(os.path.join(inc, "bvh_kernels.inc"), "w") as f:
        f.write(_kernel_part("bvh.cu", "int build_bvh("))
    with open(os.path.join(inc, "datacosts_kernels.inc"), "w") as f:
        f.write(_kernel_part("datacosts.cu", "static int finish_candidates(", ("int cub_exclusive_sum_u64", "namespace {")))
    so = os.path.join(inc, "emul_candidates.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                           "-I" + os.path.join(CPP, "emul_include"), "-I" + CPP, "-I" + CUDA_INC, "-I" + CSRC,
                           "-I" + os.path.join(ROOT, "oracle"), "-I" + inc, os.path.join(CPP, "emul_candidates.cpp"), "-o", so])
    return C.CDLL(so)


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _expected(F, fb, fe, K, nv, faces, vrank, bits, ptr, q):
    vwords = (nv + 31) // 32
    views, fids = [], []
    need = np.zeros((K, vwords), np.uint32)
    cnt = np.zeros(F + 1, np.uint64)
    for f in range(fb, fe):
        js = np.nonzero(bits[f - fb])[0]
        views.append(js); fids.append(np.full(len(js), f))
        for r in vrank[faces[f]]:
            need[js, r >> 5] |= np.uint32(1 << (int(r) & 31))
        qf = q[ptr[f]:ptr[f + 1]]
        cnt[f] = np.count_nonzero(qf != 0)   # NaN != 0 is true
    view = np.concatenate(views).astype(np.uint16) if views else np.zeros(0, np.uint16)
    face = np.concatenate(fids).astype(np.uint32) if fids else np.zeros(0, np.uint32)
    keep = q != 0
    return view, face, need, cnt, view[keep], q[keep]


@pytest.mark.parametrize("F,fb,fe,K,blocks", [(300, 0, 300, 1100, 2), (257, 40, 201, 70, 1), (64, 0, 64, 31, 3), (20, 5, 5, 40, 1)])
def test_candidate_kernels(lib, F, fb, fe, K, blocks):
    rng = np.random.RandomState(F + K)
    nv = 4 * F
    faces = rng.randint(0, nv, (F, 3)).astype(np.uint32)
    vrank = rng.permutation(nv).astype(np.uint32)
    vorder = np.argsort(vrank).astype(np.uint32)
    faces[::7, 1] = vorder[vrank[faces[::7, 0]] ^ 1]   # two vertices of the face in one bitmap word (one shared update)
    kwords = (K + 31) // 32
    bits = rng.rand(max(fe - fb, 0), K) < 0.2
    bits[::5] = False                            # faces without candidates
    words = np.zeros((max(fe - fb, 0), kwords), np.uint32)
    for j in range(K):
        words[:, j >> 5] |= (bits[:, j].astype(np.uint32) << np.uint32(j & 31))
    cnt0 = np.zeros(F + 1, np.uint64)
    cnt0[fb:fe] = bits.sum(1)
    ptr = np.concatenate([[0], np.cumsum(cnt0)[:-1]]).astype(np.uint64)   # exclusive scan over F+1 entries
    n = int(ptr[-1])
    q = rng.rand(n).astype(np.float32)
    q[rng.rand(n) < 0.3] = 0.0
    q[rng.rand(n) < 0.02] = np.nan
    view = np.zeros(max(n, 1), np.uint16)
    face = np.zeros(max(n, 1), np.uint32)
    need = np.zeros((K, (nv + 31) // 32), np.uint32)
    cnt = np.full(F + 1, 0xDEAD, np.uint64)
    dc_ptr = np.zeros(F + 1, np.uint64)
    dv = np.zeros(max(n, 1), np.uint16)
    dq = np.zeros(max(n, 1), np.float32)
    rc = lib.emul_candidate_kernels(C.c_uint32(F), C.c_uint32(fb), C.c_uint32(fe), C.c_uint32(K), C.c_uint32(nv), _p(faces), _p(vrank),
                                    _p(words), _p(ptr), _p(q if n else np.zeros(1, np.float32)), C.c_uint(blocks),
                                    _p(view), _p(face), _p(need), _p(cnt), _p(dc_ptr), _p(dv), _p(dq))
    assert rc == 0
    e_view, e_face, e_need, e_cnt, e_dv, e_dq = _expected(F, fb, fe, K, nv, faces, vrank, bits, ptr, q)
    assert np.array_equal(view[:n], e_view) and np.array_equal(face[:n], e_face)
    assert np.array_equal(need, e_need)
    assert np.array_equal(cnt, e_cnt)                 # all F+1 entries written, 0 outside [fb, fe)
    nnz = int(dc_ptr[-1])
    assert nnz == len(e_dv)
    assert np.array_equal(dv[:nnz], e_dv) and np.array_equal(dq[:nnz].view(np.uint32), e_dq.view(np.uint32))
