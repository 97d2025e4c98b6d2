"""The mesh-graph kernels of csrc/graph.cu (face adjacency, vertex -> faces, vertex -> vertices) on the serial emulator
(tests/cpp/emul_graph.cpp on tests/cpp/cuda_emul.h, kernel text unchanged), with the CUB radix sorts replaced by stable
host sorts, against scene.face_adjacency / scene.vertex_rings element for element: on the test scenes, the non-manifold
fin mesh (also against the reference's own adjacency, tests/golden/reference_tu.npz), a stress mesh with duplicate,
reversed and degenerate faces, a 40-face fan, isolated faces and unreferenced vertices, and a single face.  Small grids,
so that every thread loops over many faces.  One run of the stand-alone harness under AddressSanitizer."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import graph_meshes as GM
import refpin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mvs-texturing_b200", "csrc")
CPP = os.path.join(ROOT, "tests", "cpp")
OUT = os.path.join(CPP, "_emul", "graph")
CUDA_INC = "/usr/local/cuda/include"

pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")),
                                reason="CUDA headers not installed")


def _compile(extra, target):
    os.makedirs(OUT, exist_ok=True)
    head = open(os.path.join(CSRC, "graph.cu")).read().split("int build_mesh_graph(")[0]
    with open(os.path.join(OUT, "graph_kernels.inc"), "w") as f:
        f.write(head.replace("#include <cub/cub.cuh>", "") + "}  // namespace b2\n")
    subprocess.check_call(["/usr/bin/g++", "-O1", "-g", "-std=c++17", "-w", *extra, "-I" + CPP, "-I" + CUDA_INC,
                           "-I" + CSRC, "-I" + OUT, os.path.join(CPP, "emul_graph.cpp"), "-o", target])
    return target


@pytest.fixture(scope="module")
def lib():
    return C.CDLL(_compile(["-fPIC", "-shared"], os.path.join(OUT, "emul_graph.so")))


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _run(lib, faces, nv, blocks, threads):
    F = faces.shape[0]
    exp_adj = _host_adjacency(faces)
    cap = len(exp_adj[1]) + 16
    adj_ptr, adj_idx = np.zeros(F + 1, np.uint32), np.zeros(cap, np.uint32)
    vf_ptr, vf_idx = np.zeros(nv + 1, np.uint32), np.zeros(3 * F, np.uint32)
    vv_ptr, vv_idx = np.zeros(nv + 1, np.uint32), np.zeros(6 * F, np.uint32)
    ev, vk = np.zeros(3 * F, np.uint32), np.zeros(6 * F, np.uint64)
    stats, bad = np.zeros(4, np.uint64), np.zeros(1, np.uint64)
    faces = np.ascontiguousarray(faces, np.uint32)
    rc = lib.emul_mesh_graph(C.c_uint32(F), C.c_uint32(nv), _p(faces), C.c_uint(blocks), C.c_uint(threads), C.c_uint32(cap),
                             _p(adj_ptr), _p(adj_idx), _p(vf_ptr), _p(vf_idx), _p(vv_ptr), _p(vv_idx), _p(ev), _p(vk),
                             _p(stats), _p(bad))
    return rc, dict(adj=(adj_ptr, adj_idx[:int(stats[2])]), rings=(vf_ptr, vf_idx, vv_ptr, vv_idx[:int(stats[3])]),
                    edge_val=ev, vv_key=vk, stats=stats, bad=int(bad[0]))


def _host_adjacency(faces):
    import importlib
    return importlib.import_module("mvs-texturing_b200.scene").face_adjacency(faces)


def _meshes(scene_mod, get_scene):
    tiny = get_scene("tiny")
    out = {}
    for name in ("tiny", "messy", "occ"):
        s = scene_mod.config(name, with_images=False)
        out[name] = (s.faces, s.verts.shape[0])
    out["fins"] = GM.fin_mesh(tiny)
    out["stress"] = GM.stress_mesh(tiny)
    out["one_face"] = (np.array([[2, 0, 1]], np.uint32), 4)
    return out


def _check(scene_mod, faces, nv, r):
    ap, ai = scene_mod.face_adjacency(faces)
    rings = scene_mod.vertex_rings(faces, nv)
    assert np.array_equal(r["adj"][0], ap) and np.array_equal(r["adj"][1], ai)
    for got, want in zip(r["rings"], rings):
        assert got.dtype == want.dtype and np.array_equal(got, want)
    deg = np.diff(ap.astype(np.int64))
    assert int(r["stats"][0]) == (int(deg.max()) if len(deg) else 0)
    assert int(r["stats"][1]) == GM.non_manifold_edges(faces)


@pytest.mark.parametrize("name", ["tiny", "messy", "occ", "fins", "stress", "one_face"])
@pytest.mark.parametrize("blocks,threads", [(1, 1), (2, 32), (3, 64)])
def test_graph_kernels_match_host_arrays(lib, scene_mod, get_scene, name, blocks, threads):
    faces, nv = _meshes(scene_mod, get_scene)[name]
    rc, r = _run(lib, faces, nv, blocks, threads)
    assert rc == 0
    _check(scene_mod, faces, nv, r)


def test_fin_mesh_matches_reference_adjacency(lib, get_scene):
    faces, nv = GM.fin_mesh(get_scene("tiny"))
    rc, r = _run(lib, faces, nv, 2, 32)
    assert rc == 0
    assert int(np.diff(r["adj"][0].astype(np.int64)).max()) > 3
    assert refpin.digest(*r["adj"]) == refpin.golden()["adjacency/fins"]


def test_stress_mesh_has_every_quirk(scene_mod, get_scene):
    faces, nv = GM.stress_mesh(get_scene("tiny"))
    f = faces.astype(np.int64)
    assert ((f[:, 0] == f[:, 1]) & (f[:, 1] == f[:, 2])).any()                        # (a, a, a)
    assert ((f[:, 0] == f[:, 1]) != (f[:, 1] == f[:, 2])).any()                       # (a, a, b)
    srt = np.sort(f, 1)
    assert len(np.unique(srt, axis=0)) < len(f)                                       # duplicates
    assert int(np.diff(scene_mod.face_adjacency(faces)[0].astype(np.int64)).max()) >= 40   # the fan
    vf_ptr = scene_mod.vertex_rings(faces, nv)[0]
    assert (np.diff(vf_ptr.astype(np.int64)) == 0).sum() >= 5                         # unreferenced vertices


def test_sort_encodings_give_the_host_orders(lib, scene_mod, get_scene):
    """The kernels read the runs of the sorted edge keys as ascending by face, then by slot; the vertex -> face sort as
    np.lexsort((face, vertex)); the directed keys as np.unique of v * Vn + u."""
    faces, nv = GM.stress_mesh(get_scene("tiny"))
    rc, r = _run(lib, faces, nv, 2, 32)
    assert rc == 0
    f = faces.astype(np.int64)
    F = len(f)
    e = np.stack([f.ravel(), f[:, [1, 2, 0]].ravel()], 1)   # entry 3f+s: the edge (v_s, v_{s+1})
    lo, hi = e.min(1), e.max(1)
    fid, slot = np.repeat(np.arange(F), 3), np.tile(np.arange(3), F)
    val = r["edge_val"].astype(np.int64)
    assert np.array_equal(val, np.lexsort((slot, fid, lo * nv + hi)))
    assert np.array_equal(val, np.argsort(lo * nv + hi, kind="stable"))
    bits = max(1, int(nv - 1).bit_length())
    vk = r["vv_key"].astype(np.int64)
    dirs = np.concatenate([e, e[:, ::-1]], 0)
    assert np.array_equal(vk, np.sort(dirs[:, 0] << bits | dirs[:, 1]))
    uniq = np.unique(vk)
    assert np.array_equal((uniq >> bits) * nv + (uniq & ((1 << bits) - 1)), np.unique(dirs[:, 0] * nv + dirs[:, 1]))
    vf_order = np.lexsort((fid, f.ravel()))
    assert np.array_equal(r["rings"][1], fid[vf_order])


def test_face_index_out_of_range_is_reported(lib, get_scene):
    s = get_scene("tiny")
    faces = s.faces.copy()
    nv = s.verts.shape[0]
    faces[77, 2] = nv
    faces[150, 0] = nv + 9
    rc, r = _run(lib, faces, nv, 2, 32)
    assert rc == 1 and r["bad"] == 77


def test_graph_kernels_under_address_sanitizer(scene_mod, get_scene, tmp_path):
    exe = _compile(["-fsanitize=address", "-fno-omit-frame-pointer", "-DEMUL_GRAPH_MAIN"], os.path.join(OUT, "emul_graph_asan"))
    faces, nv = GM.stress_mesh(get_scene("tiny"))
    F = len(faces)
    ap, ai = scene_mod.face_adjacency(faces)
    src, dst = tmp_path / "in.bin", tmp_path / "out.bin"
    src.write_bytes(np.array([F, nv, 2, 32, len(ai)], np.uint32).tobytes() + faces.tobytes())
    r = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True,
                       env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0"))
    assert r.returncode == 0, r.stderr[-4000:]
    buf = dst.read_bytes()
    rc = np.frombuffer(buf, np.uint32, 1)[0]
    stats = np.frombuffer(buf, np.uint64, 4, 4)
    assert rc == 0
    rest = np.frombuffer(buf, np.uint32, offset=36)
    sizes = [F + 1, int(stats[2]), nv + 1, 3 * F, nv + 1, int(stats[3])]
    parts = np.split(rest, np.cumsum(sizes)[:-1])
    want = [ap, ai, *scene_mod.vertex_rings(faces, nv)]
    for got, w in zip(parts, want):
        assert np.array_equal(got, w)
