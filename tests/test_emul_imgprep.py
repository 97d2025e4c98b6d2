"""The batched gradient kernel k_lum_sobel of csrc/imgprep.cu on the fiber emulator (tests/cpp/emul_imgprep.cpp), bit for
bit against orc_gradient_magnitude, on view sets that the TMA kernel declines."""
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


@pytest.fixture(scope="module")
def emul():
    if not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("CUDA headers not installed")
    inc = os.path.join(OUT, "imgprep")   # own directory: the other emulation modules may hold their builds open
    os.makedirs(inc, exist_ok=True)
    text = open(os.path.join(CSRC, "imgprep.cu")).read()
    kernels = text[text.index("// ---- gradient magnitude"):text.index("// ---- TMA variant")]
    with open(os.path.join(inc, "imgprep_kernels.inc"), "w") as f:
        f.write('#include "common.cuh"\nnamespace b2 {\nnamespace {\n' + kernels + "}\n}\n")
    so = os.path.join(inc, "emul_imgprep.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                           "-I" + os.path.join(CPP, "emul_include"), "-I" + CPP, "-I" + CUDA_INC, "-I" + CSRC, "-I" + inc,
                           os.path.join(CPP, "emul_imgprep.cpp"), "-o", so])
    return C.CDLL(so)


def _p(a):
    return C.c_void_p(a.ctypes.data)


# (w, h) of one k_lum_sobel launch: the 2 x 2 and 2 x N minimum (b2tex_set_views accepts 2), odd widths and heights, views
# of one, two and three tiles (128 x 32 pixels) on each axis, and last a view whose last pixel ends the buffer
GRAD_VIEWS = [(2, 2), (2, 9), (9, 2), (3, 3), (261, 35), (48, 17), (17, 70), (2, 5), (131, 19)]


def test_k_lum_sobel_matches_the_oracle_bit_for_bit(emul, orc, scene_mod):
    """All views in one grid, packed back to back in one buffer of exactly 3 * sum(px) bytes (most views start at a byte
    that is not 4-byte aligned, and so does the buffer), with 0xFF guard bytes on both sides: every gradient pixel equals
    the oracle's, and nothing is written outside the views' gradients."""
    imgs = [np.ascontiguousarray(scene_mod.make_images(i + 1, w, h)[i]) for i, (w, h) in enumerate(GRAD_VIEWS)]
    px = np.array([w * h for w, h in GRAD_VIEWS], np.uint64)
    px_off = np.concatenate([[0], np.cumsum(px)[:-1]]).astype(np.uint64)
    total = int(px.sum())
    G = 7
    rgb_all = np.full(3 * total + 2 * G, 0xFF, np.uint8)
    rgb = rgb_all[G:G + 3 * total]
    assert total % 4 != 0 and sum((rgb.ctypes.data + 3 * int(o)) % 4 != 0 for o in px_off) >= 5
    for o, im in zip(px_off, imgs):
        rgb[3 * int(o):3 * int(o) + im.size] = im.ravel()
    grad_all = np.full(total + 2 * G, 0xAB, np.uint8)
    grad = grad_all[G:G + total]
    wh = np.array(GRAD_VIEWS, np.int32)
    assert emul.emul_gradient(C.c_uint32(len(GRAD_VIEWS)), _p(wh), _p(rgb), _p(px_off), _p(grad)) == 0
    for i, (w, h) in enumerate(GRAD_VIEWS):
        got = grad[int(px_off[i]):int(px_off[i]) + w * h].reshape(h, w)
        ref = orc.gradient_magnitude(imgs[i])
        assert np.array_equal(got, ref), (i, (w, h), int((got != ref).sum()))
    assert np.all(grad_all[:G] == 0xAB) and np.all(grad_all[G + total:] == 0xAB)
    assert grad.max() > 0
