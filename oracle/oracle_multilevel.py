"""ctypes binding of oracle/mrf_multilevel.c (oracle/_build/liborc_multilevel.so) -- TEST INFRASTRUCTURE.

Only tests/ and tools/ may import this module, like oracle.py (see oracle/oracle.h).  The product package never does.
The library is mrf_multilevel.c linked with its own copy of mrf.c (forest sampling and energies).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "liborc_multilevel.so")
# the Makefile's flags for the oracle
_CFLAGS = ["-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-fPIC", "-w"]
_SRCS = ["mrf_multilevel.c", "mrf.c"]
_DEPS = _SRCS + ["mrf_multilevel.h", "oracle.h"]


def build(force: bool = False) -> str:
    deps = [os.path.join(_HERE, f) for f in _DEPS]
    if force or not os.path.exists(_SO) or any(os.path.getmtime(d) > os.path.getmtime(_SO) for d in deps):
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        subprocess.check_call(["/usr/bin/gcc", *_CFLAGS, "-shared", "-o", _SO + ".tmp",
                               *[os.path.join(_HERE, f) for f in _SRCS], "-lm", "-Wl,--no-undefined"])
        os.replace(_SO + ".tmp", _SO)
    return _SO


class MlInfo(C.Structure):
    _fields_ = [("iterations", C.c_uint32), ("first_phase_iterations", C.c_uint32),
                ("multilevel_passes", C.c_uint32), ("coarse_nodes", C.c_uint32), ("contractions", C.c_uint32),
                ("identity_failures", C.c_uint32), ("energy_initial", C.c_double), ("energy_final", C.c_double),
                ("unseen", C.c_uint64)]


class CoarseMrf(C.Structure):
    _fields_ = [("num_nodes", C.c_uint32), ("region", C.c_void_p), ("size", C.c_void_p), ("labels", C.c_void_p),
                ("ptr", C.c_void_p), ("view", C.c_void_p), ("cost", C.c_void_p), ("cost_fixed", C.c_void_p),
                ("adj_ptr", C.c_void_p), ("adj_idx", C.c_void_p), ("weight", C.c_void_p)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
        _lib.orc_coarse_energy_fixed.restype = C.c_int64
        _lib.orc_mrf_energy_fixed.restype = C.c_int64
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def view_selection(adj_ptr, adj_idx, face_ptr, view, cost, use_multilevel=1, **kw):
    """The schedule of mrf_multilevel.c: labels, info fields, the fixed-point trace and the labels after the first
    fine phase."""
    pr = O.mrf_params(**kw)
    F = len(face_ptr) - 1
    labels = np.zeros(F, np.uint32)
    first = np.zeros(F, np.uint32)
    trace = np.full(pr.max_iterations + 1, np.nan)
    info = MlInfo()
    adj_ptr, adj_idx = np.ascontiguousarray(adj_ptr, np.uint32), np.ascontiguousarray(adj_idx, np.uint32)
    face_ptr = np.ascontiguousarray(face_ptr, np.uint64)
    view, cost = np.ascontiguousarray(view, np.uint16), np.ascontiguousarray(cost, np.float32)
    rc = lib().orc_view_selection_ml(C.c_uint32(F), _p(adj_ptr), _p(adj_idx), _p(face_ptr), _p(view), _p(cost),
                                     C.byref(pr), C.c_uint32(use_multilevel), _p(labels), _p(first), _p(trace),
                                     C.byref(info))
    if rc:
        raise RuntimeError(f"orc_view_selection_ml rc={rc}")
    r = {k: getattr(info, k) for k, _ in MlInfo._fields_}
    r.update(labels=labels, first_labels=first, trace=trace[:info.iterations + 1].copy(),
             energy=float(info.energy_final))
    return r


def contract(adj_ptr, adj_idx, face_ptr, view, cost, labels):
    """orc_mrf_contract as numpy arrays, plus the coarse fixed-point energy of the contracted labels."""
    F = len(face_ptr) - 1
    adj_ptr, adj_idx = np.ascontiguousarray(adj_ptr, np.uint32), np.ascontiguousarray(adj_idx, np.uint32)
    face_ptr = np.ascontiguousarray(face_ptr, np.uint64)
    view, cost = np.ascontiguousarray(view, np.uint16), np.ascontiguousarray(cost, np.float32)
    labels = np.ascontiguousarray(labels, np.uint32)
    c = CoarseMrf()
    L = lib()
    L.orc_mrf_contract(C.c_uint32(F), _p(adj_ptr), _p(adj_idx), _p(face_ptr), _p(view), _p(cost), _p(labels),
                       C.byref(c))
    n = int(c.num_nodes)

    def grab(ptr, ctype, count, dtype):
        if count == 0:
            return np.zeros(0, dtype)
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), (count,)).copy().astype(dtype, copy=False)
    cptr = grab(c.ptr, C.c_uint64, n + 1, np.uint64)
    cadj = grab(c.adj_ptr, C.c_uint32, n + 1, np.uint32)
    nz, ne = int(cptr[-1]), int(cadj[-1])
    out = dict(num_nodes=n, region=grab(c.region, C.c_uint32, F, np.uint32), size=grab(c.size, C.c_uint32, n, np.uint32),
               labels=grab(c.labels, C.c_uint32, n, np.uint32), ptr=cptr, view=grab(c.view, C.c_uint16, nz, np.uint16),
               cost=grab(c.cost, C.c_float, nz, np.float32), cost_fixed=grab(c.cost_fixed, C.c_int64, nz, np.int64),
               adj_ptr=cadj, adj_idx=grab(c.adj_idx, C.c_uint32, ne, np.uint32),
               weight=grab(c.weight, C.c_float, ne, np.float32))
    out["energy_fixed"] = int(L.orc_coarse_energy_fixed(C.byref(c), C.c_uint32(F), C.c_void_p(c.region)))
    L.orc_coarse_free(C.byref(c))
    return out
