"""ctypes binding of oracle/mrf_mapmap.c (oracle/_build/liborc_mapmap.so) -- TEST INFRASTRUCTURE.

Only tests/ and tools/ may import this module, like oracle.py (see oracle/oracle.h).  The product package never does.
The library is mrf_mapmap.c linked with its own copies of mrf_spanning.c, mrf_multilevel.c and mrf.c.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "liborc_mapmap.so")
# the Makefile's flags for the oracle
_CFLAGS = ["-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-fPIC", "-w"]
_SRCS = ["mrf_mapmap.c", "mrf_spanning.c", "mrf_multilevel.c", "mrf.c"]
_DEPS = _SRCS + ["mrf_mapmap.h", "mrf_spanning.h", "mrf_multilevel.h", "oracle.h"]


def build(force: bool = False) -> str:
    deps = [os.path.join(_HERE, f) for f in _DEPS]
    if force or not os.path.exists(_SO) or any(os.path.getmtime(d) > os.path.getmtime(_SO) for d in deps):
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        subprocess.check_call(["/usr/bin/gcc", *_CFLAGS, "-shared", "-o", _SO + ".tmp",
                               *[os.path.join(_HERE, f) for f in _SRCS], "-lm", "-Wl,--no-undefined"])
        os.replace(_SO + ".tmp", _SO)
    return _SO


class MmInfo(C.Structure):
    _fields_ = [("iterations", C.c_uint32), ("spanning_tree_iterations", C.c_uint32),
                ("spanning_tree_rejected", C.c_uint32), ("acyclic_iterations", C.c_uint32),
                ("multilevel_passes", C.c_uint32), ("coarse_nodes", C.c_uint32), ("multilevel_steps", C.c_uint32),
                ("multilevel_steps_rejected", C.c_uint32), ("identity_failures", C.c_uint32), ("pad", C.c_uint32),
                ("energy_initial", C.c_double), ("energy_final", C.c_double), ("unseen", C.c_uint64)]


class MmStep(C.Structure):
    _fields_ = [("num_nodes", C.c_uint32), ("rejected", C.c_uint32), ("energy_before", C.c_int64),
                ("energy_swept", C.c_int64), ("energy_after", C.c_int64), ("coarse_energy_after", C.c_int64),
                ("region", C.c_void_p), ("clabels", C.c_void_p), ("level", C.c_void_p), ("parent", C.c_void_p),
                ("swept", C.c_void_p), ("projected", C.c_void_p)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
        _lib.orc_mrf_energy_fixed.restype = C.c_int64
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _arrays(adj_ptr, adj_idx, face_ptr, view, cost):
    return [np.ascontiguousarray(adj_ptr, np.uint32), np.ascontiguousarray(adj_idx, np.uint32),
            np.ascontiguousarray(face_ptr, np.uint64), np.ascontiguousarray(view, np.uint16),
            np.ascontiguousarray(cost, np.float32)]


def view_selection(adj_ptr, adj_idx, face_ptr, view, cost, n=5, use_spanning_tree=1, use_multilevel=1, **kw):
    """The schedule of mrf_mapmap.c (n = spanning_tree_multilevel_after_n_iterations): labels, info fields and the
    fixed-point trace.  Raises ValueError for the argument error (rc 2)."""
    pr = O.mrf_params(**kw)
    F = len(face_ptr) - 1
    labels = np.zeros(F, np.uint32)
    trace = np.full(pr.max_iterations + 1, np.nan)
    info = MmInfo()
    ap, ai, fp, view, cost = _arrays(adj_ptr, adj_idx, face_ptr, view, cost)
    rc = lib().orc_view_selection_mapmap(C.c_uint32(F), _p(ap), _p(ai), _p(fp), _p(view), _p(cost), C.byref(pr),
                                         C.c_uint32(use_spanning_tree), C.c_uint32(use_multilevel), C.c_uint32(n),
                                         _p(labels), _p(trace), C.byref(info))
    if rc == 2:
        raise ValueError("spanning_tree_multilevel_after_n_iterations > 0 needs use_spanning_tree and use_multilevel")
    if rc:
        raise RuntimeError(f"orc_view_selection_mapmap rc={rc}")
    r = {k: getattr(info, k) for k, _ in MmInfo._fields_ if k != "pad"}
    r.update(labels=labels, trace=trace[:info.iterations + 1].copy(), energy=float(info.energy_final))
    return r


def step(adj_ptr, adj_idx, face_ptr, view, cost, labels, iteration, **kw):
    """one multilevel step from `labels`: dict(labels (after acceptance), region, clabels, level, parent, swept,
    projected, num_nodes, rejected, energies)"""
    pr = O.mrf_params(**kw)
    F = len(face_ptr) - 1
    ap, ai, fp, view, cost = _arrays(adj_ptr, adj_idx, face_ptr, view, cost)
    out = np.array(labels, np.uint32)
    arr = {k: np.zeros(max(F, 1), np.uint32) for k in ("region", "clabels", "level", "parent", "swept", "projected")}
    st = MmStep()
    for k, a in arr.items():
        setattr(st, k, a.ctypes.data)
    lib().orc_mrf_mapmap_step(C.c_uint32(F), _p(ap), _p(ai), _p(fp), _p(view), _p(cost), C.byref(pr),
                              C.c_uint32(iteration), _p(out), C.byref(st))
    n = st.num_nodes
    r = dict(labels=out, num_nodes=n, rejected=bool(st.rejected), energy_before=st.energy_before,
             energy_swept=st.energy_swept, energy_after=st.energy_after, coarse_energy_after=st.coarse_energy_after)
    r.update(region=arr["region"][:F], projected=arr["projected"][:F])
    r.update({k: arr[k][:n].copy() for k in ("clabels", "level", "parent", "swept")})
    return r


def spanning_sweep(adj_ptr, adj_idx, face_ptr, view, cost, labels, iteration, weight=None, **kw):
    """the weighted spanning DP of one iteration (no acceptance): (labels after the DP, level, parent)"""
    pr = O.mrf_params(**kw)
    F = len(face_ptr) - 1
    ap, ai, fp, view, cost = _arrays(adj_ptr, adj_idx, face_ptr, view, cost)
    w = None if weight is None else np.ascontiguousarray(weight, np.float32)
    out = np.array(labels, np.uint32)
    level, parent = np.zeros(F, np.uint32), np.zeros(F, np.uint32)
    lib().orc_mrf_spanning_sweep_w(C.c_uint32(F), _p(ap), _p(ai), _p(w) if w is not None else None, _p(fp), _p(view),
                                   _p(cost), C.byref(pr), C.c_uint32(iteration), _p(out), _p(level), _p(parent))
    return out, level, parent
