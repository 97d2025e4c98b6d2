"""ctypes binding of oracle/mrf_spanning.c (oracle/_build/liborc_spanning.so) -- TEST INFRASTRUCTURE.

Only tests/ and tools/ may import this module, like oracle.py (see oracle/oracle.h).  The product package never does.
The library is mrf_spanning.c linked with its own copies of mrf_multilevel.c and mrf.c.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "liborc_spanning.so")
# the Makefile's flags for the oracle
_CFLAGS = ["-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-fPIC", "-w"]
_SRCS = ["mrf_spanning.c", "mrf_multilevel.c", "mrf.c"]
_DEPS = _SRCS + ["mrf_spanning.h", "mrf_multilevel.h", "oracle.h"]


def build(force: bool = False) -> str:
    deps = [os.path.join(_HERE, f) for f in _DEPS]
    if force or not os.path.exists(_SO) or any(os.path.getmtime(d) > os.path.getmtime(_SO) for d in deps):
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        subprocess.check_call(["/usr/bin/gcc", *_CFLAGS, "-shared", "-o", _SO + ".tmp",
                               *[os.path.join(_HERE, f) for f in _SRCS], "-lm", "-Wl,--no-undefined"])
        os.replace(_SO + ".tmp", _SO)
    return _SO


class StInfo(C.Structure):
    _fields_ = [("iterations", C.c_uint32), ("spanning_tree_iterations", C.c_uint32),
                ("spanning_tree_rejected", C.c_uint32), ("acyclic_iterations", C.c_uint32),
                ("multilevel_passes", C.c_uint32), ("coarse_nodes", C.c_uint32), ("energy_initial", C.c_double),
                ("energy_final", C.c_double), ("unseen", C.c_uint64)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
        _lib.orc_mrf_sample_spanning.restype = C.c_uint32
        _lib.orc_mrf_energy_fixed.restype = C.c_int64
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _arrays(adj_ptr, adj_idx, face_ptr, view=None, cost=None):
    out = [np.ascontiguousarray(adj_ptr, np.uint32), np.ascontiguousarray(adj_idx, np.uint32),
           np.ascontiguousarray(face_ptr, np.uint64)]
    if view is not None:
        out += [np.ascontiguousarray(view, np.uint16), np.ascontiguousarray(cost, np.float32)]
    return out


def view_selection(adj_ptr, adj_idx, face_ptr, view, cost, use_spanning_tree=1, use_multilevel=0, **kw):
    """The schedule of mrf_spanning.c: labels, info fields and the fixed-point trace."""
    pr = O.mrf_params(**kw)
    F = len(face_ptr) - 1
    labels = np.zeros(F, np.uint32)
    trace = np.full(pr.max_iterations + 1, np.nan)
    info = StInfo()
    ap, ai, fp, view, cost = _arrays(adj_ptr, adj_idx, face_ptr, view, cost)
    rc = lib().orc_view_selection_st(C.c_uint32(F), _p(ap), _p(ai), _p(fp), _p(view), _p(cost), C.byref(pr),
                                     C.c_uint32(use_spanning_tree), C.c_uint32(use_multilevel), _p(labels), _p(trace),
                                     C.byref(info))
    if rc:
        raise RuntimeError(f"orc_view_selection_st rc={rc}")
    r = {k: getattr(info, k) for k, _ in StInfo._fields_}
    r.update(labels=labels, trace=trace[:info.iterations + 1].copy(), energy=float(info.energy_final))
    return r


def sample_spanning(adj_ptr, adj_idx, face_ptr, iteration, **kw):
    """(level, parent, deepest level) of the spanning forest of one iteration"""
    pr = O.mrf_params(**kw)
    F = len(face_ptr) - 1
    ap, ai, fp = _arrays(adj_ptr, adj_idx, face_ptr)
    level, parent = np.zeros(F, np.uint32), np.zeros(F, np.uint32)
    depth = lib().orc_mrf_sample_spanning(C.c_uint32(F), _p(ap), _p(ai), _p(fp), C.byref(pr), C.c_uint32(iteration),
                                          _p(level), _p(parent))
    return level, parent, int(depth)


def spanning_iteration(adj_ptr, adj_idx, face_ptr, view, cost, labels, iteration, **kw):
    """one spanning iteration from `labels`: dict(labels (after acceptance), swept (before), level, parent, rejected)"""
    pr = O.mrf_params(**kw)
    F = len(face_ptr) - 1
    ap, ai, fp, view, cost = _arrays(adj_ptr, adj_idx, face_ptr, view, cost)
    out = np.array(labels, np.uint32)
    swept, level, parent = np.zeros(F, np.uint32), np.zeros(F, np.uint32), np.zeros(F, np.uint32)
    rej = lib().orc_mrf_spanning_iteration(C.c_uint32(F), _p(ap), _p(ai), _p(fp), _p(view), _p(cost), C.byref(pr),
                                           C.c_uint32(iteration), _p(out), _p(level), _p(parent), _p(swept))
    return dict(labels=out, swept=swept, level=level, parent=parent, rejected=bool(rej))
