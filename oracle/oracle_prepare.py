"""ctypes binding of oracle/prepare_mesh.c (oracle/_build/liborc_prepare.so) -- TEST INFRASTRUCTURE.

Only tests/ and tools/ may import this module, like oracle.py (see oracle/oracle.h).  The product package never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "liborc_prepare.so")
# the Makefile's flags for the oracle
_CFLAGS = ["-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-w"]


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "prepare_mesh.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(src) > os.path.getmtime(_SO):
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        subprocess.check_call(["/usr/bin/gcc", *_CFLAGS, "-shared", "-o", _SO + ".tmp", src, "-lm", "-Wl,--no-undefined"])
        os.replace(_SO + ".tmp", _SO)
    return _SO


_REF_SO = os.path.join(_HERE, "_ref", "libprepref.so")
REFERENCE = os.environ.get("B2TEX_REFERENCE", "")


def build_ref() -> str | None:
    """The reference's own prepare_mesh.cpp (unmodified, compiled where it lies) with ref_prepare_glue.cpp against the
    shims refshim_prepare + refshim, into oracle/_ref/libprepref.so -- only where B2TEX_REFERENCE names a checkout of the
    reference; otherwise a prebuilt library is used as is.  tests/golden/make_prepare_mesh_golden.py reads it."""
    src = os.path.join(REFERENCE, "libs", "tex", "prepare_mesh.cpp")
    if REFERENCE and os.path.exists(src):
        deps = [src, os.path.join(_HERE, "ref_prepare_glue.cpp"), os.path.join(_HERE, "refshim_prepare", "mve", "mesh.h")]
        if not os.path.exists(_REF_SO) or any(os.path.getmtime(d) > os.path.getmtime(_REF_SO) for d in deps):
            os.makedirs(os.path.dirname(_REF_SO), exist_ok=True)
            # the Makefile's flags for the reference TUs
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++11", "-march=x86-64-v3", "-ffp-contract=off",
                                   "-fno-fast-math", "-fopenmp", "-fPIC", "-w", "-shared", "-o", _REF_SO + ".tmp",
                                   "-I" + os.path.join(_HERE, "refshim_prepare"), "-I" + _HERE,
                                   "-I" + os.path.join(_HERE, "refshim"), "-I" + os.path.join(REFERENCE, "libs"),
                                   os.path.join(_HERE, "ref_prepare_glue.cpp"), src, "-lm"])
            os.replace(_REF_SO + ".tmp", _REF_SO)
    return _REF_SO if os.path.exists(_REF_SO) else None


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
        for fn in ("orc_remove_redundant_faces", "orc_face_normals"):
            getattr(_lib, fn).restype = C.c_uint32
    return _lib


def _p(a):
    return C.c_void_p(a.ctypes.data)


def remove_redundant_faces(faces, num_verts):
    """(kept faces u32[F', 3], kept input ids u32[F'], number removed), prepare_mesh.cpp:14-55"""
    f = np.ascontiguousarray(faces, np.uint32).reshape(-1, 3)
    keep = np.zeros(len(f), np.uint8)
    n = lib().orc_remove_redundant_faces(_p(f), C.c_uint32(len(f)), C.c_uint32(num_verts), _p(keep))
    kept = np.flatnonzero(keep).astype(np.uint32)
    return np.ascontiguousarray(f[kept]), kept, int(n)


def face_normals(verts, faces):
    """(normals f32[F, 3], number of zero normals)"""
    v, f = np.ascontiguousarray(verts, np.float32), np.ascontiguousarray(faces, np.uint32).reshape(-1, 3)
    out = np.empty((len(f), 3), np.float32)
    z = lib().orc_face_normals(_p(v), _p(f), C.c_uint32(len(f)), _p(out))
    return out, int(z)


def vertex_normals(verts, faces):
    v, f = np.ascontiguousarray(verts, np.float32), np.ascontiguousarray(faces, np.uint32).reshape(-1, 3)
    out = np.empty((len(v), 3), np.float32)
    lib().orc_vertex_normals(_p(v), C.c_uint32(len(v)), _p(f), C.c_uint32(len(f)), _p(out))
    return out


def prepare_mesh(verts, faces):
    """everything b2tex_prepare_mesh computes: dict(faces, kept, num_redundant, face_normals, num_zero_normals,
    vertex_normals)"""
    v = np.ascontiguousarray(verts, np.float32)
    kf, kept, n = remove_redundant_faces(faces, len(v))
    fn, z = face_normals(v, kf)
    return dict(faces=kf, kept=kept, num_redundant=n, face_normals=fn, num_zero_normals=z,
                vertex_normals=vertex_normals(v, kf))
