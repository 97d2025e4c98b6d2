"""ctypes binding of oracle/undistort.c (oracle/_build/liborc_undistort.so) -- TEST INFRASTRUCTURE.

Only tests/ and tools/ may import this module, like oracle.py (see oracle/oracle.h).  The product package never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "liborc_undistort.so")
# the Makefile's flags for the oracle
_CFLAGS = ["-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-fPIC", "-w"]


def build(force: bool = False) -> str:
    srcs = [os.path.join(_HERE, f) for f in ("undistort.c", "datacosts.c", "bvh.c", "imgprep.c", "oracle.h")]
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        subprocess.check_call(["/usr/bin/gcc", *_CFLAGS, "-shared", "-o", _SO + ".tmp", os.path.join(_HERE, "undistort.c"),
                               # what datacosts.c calls: the BVH of its visibility rays, the image preparation
                               os.path.join(_HERE, "bvh.c"), os.path.join(_HERE, "imgprep.c"), "-lm", "-Wl,--no-undefined"])
        os.replace(_SO + ".tmp", _SO)
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
    return _lib


def undistort(rgb, flen, k0, k1=0.0):
    """The (H, W, 3) u8 image of a .cam view as texturing sees it (orc_undistort)."""
    h, w, _ = rgb.shape
    src = np.ascontiguousarray(rgb, np.uint8)
    out = np.empty_like(src)
    lib().orc_undistort(src.ctypes.data_as(C.c_void_p), w, h, C.c_float(flen), C.c_float(k0), C.c_float(k1),
                        out.ctypes.data_as(C.c_void_p))
    return out
