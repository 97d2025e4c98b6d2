"""Undistortion on the CPU: properties of the oracle's restatement of MVE's two models (oracle/undistort.c), k_undistort of
csrc/undistort.cu on the host emulator bit for bit against it, and the batched validity flood of csrc/imgprep.cu on the
fiber emulator against orc_validity_mask (tests/cpp/emul_undistort.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_undistort as ou   # oracle/ is on sys.path (tests/conftest.py)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mvs-texturing_b200", "csrc")
CPP = os.path.join(ROOT, "tests", "cpp")
OUT = os.path.join(CPP, "_emul")
CUDA_INC = "/usr/local/cuda/include"


def _images(scene_mod, sizes):
    """one make_images view per (w, h): every channel >= 1, so a zero pixel can only be zero fill"""
    return [np.ascontiguousarray(scene_mod.make_images(i + 1, w, h)[i]) for i, (w, h) in enumerate(sizes)]


def _bilinear(img, sx, sy):
    """float bilinear sample (edge clamped) of an (H, W, 3) image at index positions"""
    h, w, _ = img.shape
    x = np.clip(sx, 0, w - 1)
    y = np.clip(sy, 0, h - 1)
    x0 = np.floor(x).astype(int)
    y0 = np.floor(y).astype(int)
    x1, y1 = np.minimum(x0 + 1, w - 1), np.minimum(y0 + 1, h - 1)
    fx, fy = (x - x0)[..., None], (y - y0)[..., None]
    f = img.astype(np.float64)
    return (f[y0, x0] * (1 - fx) * (1 - fy) + f[y0, x1] * fx * (1 - fy) + f[y1, x0] * (1 - fx) * fy + f[y1, x1] * fx * fy)


def _centred(w, h, fl):
    x = (np.arange(w, dtype=np.float64)[None, :] + 0.5 - 0.5 * w) / fl
    y = (np.arange(h, dtype=np.float64)[:, None] + 0.5 - 0.5 * h) / fl
    return np.broadcast_to(x, (h, w)), np.broadcast_to(y, (h, w))


def _source(w, h, flen, k0, k1):
    """The source position oracle/undistort.c documents, with its arithmetic: (px, py) continuous, NaN where there is none."""
    fl = np.float64(np.float32(flen)) * max(w, h)
    k0, k1 = np.float64(np.float32(k0)), np.float64(np.float32(k1))
    ux, uy = _centred(w, h, fl)
    r2 = ux * ux + uy * uy
    if k1 != 0:
        s = 1.0 + k0 * r2 + k1 * r2 * r2
    else:
        q = k0 * r2
        s = np.ones_like(q)
        active = np.ones(q.shape, bool)
        for _ in range(100):
            sn = s - (q * s * s * s + s - 1.0) / (3.0 * q * s * s + 1.0)
            done = sn == s
            s = np.where(active, sn, s)
            active &= ~done
            if not active.any():
                break
        s = np.where(27.0 * q < -4.0, np.nan, s)
    return ux * s * fl + 0.5 * w, uy * s * fl + 0.5 * h


def _distort(img, flen, k0, k1):
    """The forward models (a distorted image from an undistorted one), float bilinear; NaN where undefined.
    VisualSFM in closed form (undistorted = distorted (1 + k r_d^2)); Bundler by Newton on the radius."""
    h, w, _ = img.shape
    fl = float(np.float32(flen)) * max(w, h)
    dx, dy = _centred(w, h, fl)
    rd2 = dx * dx + dy * dy
    if k1 != 0:
        rd = np.sqrt(rd2)
        ru = rd.copy()
        for _ in range(50):
            ru = ru - (ru * (1 + k0 * ru ** 2 + k1 * ru ** 4) - rd) / (1 + 3 * k0 * ru ** 2 + 5 * k1 * ru ** 4)
        scale = np.where(rd > 0, ru / np.where(rd > 0, rd, 1), 1.0)
    else:
        scale = 1.0 + k0 * rd2
    px, py = dx * scale * fl + 0.5 * w, dy * scale * fl + 0.5 * h
    out = _bilinear(img, px - 0.5, py - 0.5)
    inside = (px >= 0) & (px < w) & (py >= 0) & (py < h)
    out[~inside] = np.nan
    return out


# ---- oracle properties (independent of how MVE words the models) -------------------------------------------------
def test_zero_distortion_is_a_copy(scene_mod):
    img = _images(scene_mod, [(61, 37)])[0]
    for k in [(0.0, 0.0), (0.0, 0.3), (0.0, -0.2)]:
        assert np.array_equal(ou.undistort(img, 0.9, *k), img), k


@pytest.mark.parametrize("flen,k0,k1", [(1.0, 0.08, 0.0), (1.0, -0.08, 0.0), (0.9, 0.1, 0.02), (0.9, -0.1, 0.02)])
def test_round_trip_through_the_forward_model(scene_mod, flen, k0, k1):
    """Distort a view with the forward model, undistort it: inside the region where both maps are defined (2 px away
    from the image border) the result is the original within two bilinear resamplings of a band-limited texture."""
    img = _images(scene_mod, [(240, 180)])[0]
    h, w, _ = img.shape
    dist = _distort(img, flen, k0, k1)
    defined = ~np.isnan(dist[..., 0])
    dist_u8 = np.where(np.isnan(dist), 0, np.floor(np.nan_to_num(dist) + 0.5)).astype(np.uint8)
    back = ou.undistort(dist_u8, flen, k0, k1).astype(np.int32)
    px, py = _source(w, h, flen, k0, k1)
    sx, sy = px - 0.5, py - 0.5
    ok = (sx >= 2) & (sx <= w - 3) & (sy >= 2) & (sy <= h - 3)
    # the four distorted pixels around the source must all be defined
    x0 = np.clip(np.floor(np.nan_to_num(sx)).astype(int), 0, w - 2)
    y0 = np.clip(np.floor(np.nan_to_num(sy)).astype(int), 0, h - 2)
    ok &= defined[y0, x0] & defined[y0, x0 + 1] & defined[y0 + 1, x0] & defined[y0 + 1, x0 + 1]
    assert ok.mean() > 0.6
    err = np.abs(back - img.astype(np.int32))[ok]
    assert err.mean() < 2.5 and np.percentile(err, 99) <= 12, (err.mean(), np.percentile(err, 99), err.max())


@pytest.mark.parametrize("flen,k0,k1", [(0.8, 0.25, 0.0), (0.5, -0.9, 0.0), (0.7, 0.3, 0.1), (0.7, -0.15, 0.05),
                                        (1.1, -0.05, 0.0), (1.0, 0.05, 0.0)])
def test_zero_fill_is_where_the_source_leaves_the_image(scene_mod, flen, k0, k1):
    """(0.5, -0.9): VisualSFM's cubic has no positive root in the corners; (1.1, -0.05), (1.0, 0.05): sources stay inside."""
    img = _images(scene_mod, [(97, 66)])[0]
    h, w, _ = img.shape
    out = ou.undistort(img, flen, k0, k1)
    px, py = _source(w, h, flen, k0, k1)
    outside = ~((px >= 0) & (px < w) & (py >= 0) & (py < h))   # NaN compares false: no source
    zero = (out == 0).all(-1)
    assert np.array_equal(zero, outside)
    assert np.all(out[~outside] > 0)
    if (flen, k0) == (0.5, -0.9):
        assert np.isnan(px).any()


# ---- emulation ----------------------------------------------------------------------------------------------------
def _kernel_text(cu_file, begin=None, end=None):
    text = open(os.path.join(CSRC, cu_file)).read()
    a = text.index(begin) if begin else 0
    b = text.index(end)
    return text[a:b]


@pytest.fixture(scope="module")
def emul():
    if not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("CUDA headers not installed")
    inc = os.path.join(OUT, "undistort")   # own directory: the other emulation modules may hold their builds open
    os.makedirs(inc, exist_ok=True)
    with open(os.path.join(inc, "undistort_kernels.inc"), "w") as f:
        f.write(_kernel_text("undistort.cu", end="// Scratch for one batch") + "}  // namespace b2\n")
    with open(os.path.join(inc, "flood_kernels.inc"), "w") as f:
        f.write('#include "common.cuh"\nnamespace b2 {\nnamespace {\n'
                + _kernel_text("imgprep.cu", "// one view of a batched flood", "// erosion (optional)") + "}\n}\n")
    so = os.path.join(inc, "emul_undistort.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w",
                           "-I" + os.path.join(CPP, "emul_include"), "-I" + CPP, "-I" + CUDA_INC, "-I" + CSRC, "-I" + inc,
                           os.path.join(CPP, "emul_undistort.cpp"), "-o", so])
    return C.CDLL(so)


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _pack(imgs, align):
    offs, pos = [], 0
    for im in imgs:
        offs.append(pos)
        pos += (im.size + align - 1) // align * align
    buf = np.zeros(max(pos, 1), np.uint8)
    for o, im in zip(offs, imgs):
        buf[o:o + im.size] = im.ravel()
    return buf, np.array(offs, np.uint64)


# (w, h, flen, k0, k1): odd widths, mixed sizes, both models, black borders and none, a VisualSFM case without a root
EMUL_VIEWS = [(37, 23, 0.8, 0.25, 0.0), (64, 48, 0.9, 0.2, 0.05), (50, 31, 0.5, -0.9, 0.0), (33, 40, 1.0, 0.04, 0.0),
              (45, 45, 1.2, -0.1, 0.01), (70, 19, 0.7, -0.3, 0.08), (18, 26, 1.0, -0.05, 0.0)]


def test_k_undistort_matches_the_oracle_bit_for_bit(emul, scene_mod):
    imgs = _images(scene_mod, [(v[0], v[1]) for v in EMUL_VIEWS])
    src, src_off = _pack(imgs, 3)
    dst, dst_off = _pack(imgs, 16)
    dst[:] = 0xAB
    wh = np.array([[v[0], v[1]] for v in EMUL_VIEWS], np.int32)
    flen = np.array([v[2] for v in EMUL_VIEWS], np.float32)
    k = np.array([[v[3], v[4]] for v in EMUL_VIEWS], np.float32)
    assert emul.emul_undistort(C.c_uint32(len(EMUL_VIEWS)), _p(wh), _p(src), _p(src_off), _p(dst), _p(dst_off), _p(flen), _p(k)) == 0
    black = 0
    for i, (w, h, fl, k0, k1) in enumerate(EMUL_VIEWS):
        got = dst[int(dst_off[i]):int(dst_off[i]) + 3 * w * h].reshape(h, w, 3)
        ref = ou.undistort(imgs[i], fl, k0, k1)
        assert np.array_equal(got, ref), (i, int((got != ref).any(-1).sum()))
        black += bool((ref == 0).all(-1).any())
        tail = dst[int(dst_off[i]) + 3 * w * h:int(dst_off[i + 1]) if i + 1 < len(EMUL_VIEWS) else len(dst)]
        assert np.all(tail == 0xAB)   # nothing written past a view
    assert 0 < black < len(EMUL_VIEWS)


def test_batched_flood_matches_the_oracle_masks(emul, orc, scene_mod):
    """several flagged views of different sizes flooded in the same rounds (one k_flood grid over all of them)"""
    sizes = [(70, 45), (33, 66), (97, 40), (40, 40)]
    imgs = _images(scene_mod, sizes)
    imgs[0][:9] = 0; imgs[0][:, :5] = 0; imgs[0][20:25, 30:40] = 0              # border + an interior blob
    imgs[1][-3:, -40:] = 0; imgs[1][:, -2:] = 0                                 # bottom-right corner region
    imgs[2] = ou.undistort(imgs[2], 0.6, 0.3, 0.05)                             # zero fill of a pincushion undistortion
    imgs[3][0, :] = 0; imgs[3][:30, 19:21] = 0                                  # top row and a wall hanging from it
    src, off = _pack(imgs, 3)
    px_off = (off // 3).astype(np.uint64)
    wh = np.array(sizes, np.int32)
    inv = np.full(sum(w * h for w, h in sizes), 7, np.uint8)
    rounds = emul.emul_flood(C.c_uint32(len(sizes)), _p(wh), _p(src), _p(px_off), _p(inv))
    assert rounds > 1
    for i, (w, h) in enumerate(sizes):
        got = inv[int(px_off[i]):int(px_off[i]) + w * h].reshape(h, w)
        ref = orc.validity_mask(imgs[i]) == 0
        assert ref.any()
        assert np.array_equal(got.astype(bool), ref), (i, int((got.astype(bool) != ref).sum()))
