"""The mesh-preparation kernels of csrc/prepare.cu after the sorts (sets, runs, degenerate-set table, subset lookups,
compaction with face normals, vertex normals) on the serial emulator (tests/cpp/emul_prepare.cpp on tests/cpp/cuda_emul.h,
kernel text unchanged), with the CUB radix sorts replaced by stable host sorts, against the ring-scan oracle
(oracle/prepare_mesh.c) on the meshes of tests/test_prepare_mesh_cpu.py.  Both sort forms (one 64-bit pass, two passes)
give the same order; vertex ids >= 2^22 take the two-pass form by themselves.  Small grids, so that every thread loops
over many faces.  One run of the stand-alone harness under AddressSanitizer."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_prepare as OP
from test_prepare_mesh_cpu import MESHES, quirk_mesh, prep_meshes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mvs-texturing_b200", "csrc")
CPP = os.path.join(ROOT, "tests", "cpp")
OUT = os.path.join(CPP, "_emul", "prepare")
CUDA_INC = "/usr/local/cuda/include"

pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")),
                                reason="CUDA headers not installed")


def _compile(extra, target):
    os.makedirs(OUT, exist_ok=True)
    head = open(os.path.join(CSRC, "prepare.cu")).read().split("int prepare_mesh(")[0]
    with open(os.path.join(OUT, "prepare_kernels.inc"), "w") as f:
        f.write(head.replace("#include <cub/cub.cuh>", "") + "}  // namespace b2\n")
    subprocess.check_call(["/usr/bin/g++", "-O1", "-g", "-std=c++17", "-w", "-ffp-contract=off", *extra, "-I" + CPP,
                           "-I" + CUDA_INC, "-I" + CSRC, "-I" + OUT, os.path.join(CPP, "emul_prepare.cpp"), "-o", target])
    return target


@pytest.fixture(scope="module")
def lib():
    return C.CDLL(_compile(["-fPIC", "-shared"], os.path.join(OUT, "emul_prepare.so")))


@pytest.fixture(scope="module")
def meshes(scene_mod, get_scene):
    m = prep_meshes(scene_mod, get_scene("tiny"))
    m["wide"] = quirk_mesh(5, offset=(1 << 22) + 37)   # 23-bit vertex ids: 69-bit sets
    return m


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _run(lib, verts, faces, wide=0, blocks=2, threads=32):
    F, nv = len(faces), len(verts)
    faces = np.ascontiguousarray(faces, np.uint32)
    verts = np.ascontiguousarray(verts, np.float32)
    of, kept, nrm = np.zeros((F, 3), np.uint32), np.zeros(F, np.uint32), np.zeros((F, 3), np.float32)
    srt, stats = np.zeros(F, np.uint32), np.zeros(4, np.uint64)
    rc = lib.emul_prepare_faces(C.c_uint32(F), C.c_uint32(nv), _p(faces), _p(verts), C.c_int(wide), C.c_uint(blocks),
                                C.c_uint(threads), _p(of), _p(kept), _p(nrm), _p(srt), _p(stats))
    Fk = int(stats[0])
    return rc, dict(faces=of[:Fk], kept=kept[:Fk], face_normals=nrm[:Fk], sorted=srt, table=int(stats[1]),
                    zeros=int(stats[2]), narrow=bool(stats[3]))


def _set_order(faces):
    s = np.sort(faces.astype(np.int64), 1)
    s[:, 1] = np.where(s[:, 0] == s[:, 1], s[:, 2], s[:, 1])   # distinct members, padded with the largest
    return np.lexsort((np.arange(len(s)), s[:, 2], s[:, 1], s[:, 0])), s


@pytest.mark.parametrize("name", MESHES + ("wide",))
@pytest.mark.parametrize("blocks,threads", [(1, 1), (2, 32), (3, 64)])
def test_kernels_match_the_ring_scan_oracle(lib, meshes, name, blocks, threads):
    verts, faces = meshes[name]
    rc, r = _run(lib, verts, faces, 0, blocks, threads)
    assert rc == 0
    o = OP.prepare_mesh(verts, faces)
    assert np.array_equal(r["faces"], o["faces"]) and np.array_equal(r["kept"], o["kept"])
    assert len(faces) - len(r["kept"]) == o["num_redundant"]
    assert np.array_equal(r["face_normals"].view(np.uint32), o["face_normals"].view(np.uint32))
    assert r["zeros"] == o["num_zero_normals"]
    assert r["narrow"] == (name != "wide")


@pytest.mark.parametrize("name", ["stress", "quirk0", "wide"])
def test_both_sort_forms_give_the_set_order(lib, meshes, name):
    verts, faces = meshes[name]
    order, s = _set_order(faces)
    runs = []
    for wide in (0, 1):
        if name == "wide" and not wide:
            continue
        rc, r = _run(lib, verts, faces, wide)
        assert rc == 0 and r["narrow"] == (not wide)
        assert np.array_equal(r["sorted"], order)
        assert r["table"] == len(np.unique(s[s[:, 1] == s[:, 2]], axis=0))
        runs.append(r)
    if len(runs) == 2:
        assert all(np.array_equal(runs[0][k], runs[1][k]) for k in ("faces", "kept", "face_normals"))


def test_clean_mesh_skips_the_table(lib, meshes):
    verts, faces = meshes["occ"]
    rc, r = _run(lib, verts, faces)
    assert rc == 0 and r["table"] == 0 and np.array_equal(r["faces"], faces)


@pytest.mark.parametrize("name", MESHES)
def test_vertex_normals_match_the_oracle_bit_for_bit(lib, scene_mod, meshes, name):
    """Same libm acosf on both sides here, so the face-loop oracle and the vertex-row kernel must agree exactly: the
    order of the sums is the same."""
    verts, faces = meshes[name]
    o = OP.prepare_mesh(verts, faces)
    kf = np.ascontiguousarray(o["faces"], np.uint32)
    vf_ptr, vf_idx, _, _ = scene_mod.vertex_rings(kf, len(verts))
    vn = np.zeros((len(verts), 3), np.float32)
    v = np.ascontiguousarray(verts, np.float32)
    lib.emul_vertex_normals(C.c_uint32(len(verts)), _p(v), _p(kf), _p(np.ascontiguousarray(vf_ptr)),
                            _p(np.ascontiguousarray(vf_idx)), C.c_uint(3), C.c_uint(64), _p(vn))
    assert np.array_equal(vn.view(np.uint32), o["vertex_normals"].view(np.uint32))


def test_kernels_under_address_sanitizer(meshes, tmp_path):
    exe = _compile(["-fsanitize=address", "-fno-omit-frame-pointer", "-DEMUL_PREPARE_MAIN"],
                   os.path.join(OUT, "emul_prepare_asan"))
    for name, wide in (("stress", 0), ("quirk1", 1)):
        verts, faces = meshes[name]
        F, nv = len(faces), len(verts)
        src, dst = tmp_path / "in.bin", tmp_path / "out.bin"
        src.write_bytes(np.array([F, nv, wide, 2, 32], np.uint32).tobytes() + np.ascontiguousarray(faces, np.uint32).tobytes()
                        + np.ascontiguousarray(verts, np.float32).tobytes())
        r = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True,
                           env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0"))
        assert r.returncode == 0, r.stderr[-4000:]
        buf = dst.read_bytes()
        assert np.frombuffer(buf, np.uint32, 1)[0] == 0
        Fk = int(np.frombuffer(buf, np.uint64, 1, 4)[0])
        rest = np.frombuffer(buf, np.uint32, offset=36)
        o = OP.prepare_mesh(verts, faces)
        assert np.array_equal(rest[:3 * Fk].reshape(-1, 3), o["faces"])
        assert np.array_equal(rest[3 * Fk:4 * Fk], o["kept"])
        assert np.array_equal(rest[4 * Fk:7 * Fk], o["face_normals"].view(np.uint32).ravel())
