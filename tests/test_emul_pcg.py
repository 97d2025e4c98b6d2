"""k_pcg (csrc/seam.cu) under the fiber emulator on hand-built systems, bit for bit against tests/golden/pcg_emul.npz.

The golden file holds what an earlier k_pcg computed (the commit is stored in it; tests/golden/make_pcg_emul.py).  The
systems cover a pair loop with a tail (R not a multiple of 2 x 1024), threads that own several row pairs, rows with
only a (possibly zero) diagonal, a row longer than the SpMV's register batch, both weight classes, a channel with a
zero right-hand side, channels that stop in different iterations and a solve that stops at max_iters.  Any change
of operand or summation order in the solve shows up here as a changed bit.
"""
import importlib.util
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "cpp", "_emul", "pcg")

pytestmark = pytest.mark.skipif(not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"), reason="CUDA headers not installed")

_spec = importlib.util.spec_from_file_location("make_pcg_emul", os.path.join(ROOT, "tests", "golden", "make_pcg_emul.py"))
gen = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gen)


@pytest.fixture(scope="module")
def lib():
    with open(os.path.join(ROOT, "mvs-texturing_b200", "csrc", "seam.cu")) as f:
        return gen.build(f.read(), OUT)


@pytest.fixture(scope="module")
def golden():
    return np.load(gen.GOLDEN)


@pytest.mark.parametrize("name", list(gen.SYSTEMS))
def test_pcg_iterates_bit_identical(lib, golden, name):
    R, seed, zc, mi = gen.SYSTEMS[name]
    sysd = gen.make_system(R, seed, zero_rhs_channel=zc)
    assert int(np.diff(sysd["ptr"]).max()) >= 40 and (sysd["diag"] == 0).any()
    st, x = gen.run(lib, sysd, mi)
    ref_st, ref_x = golden[name + "/status"], golden[name + "/x"]
    assert st.tolist() == ref_st.tolist(), f"iterations / residual bits / loops differ from {golden['commit']}"
    assert np.array_equal(x.view(np.uint32), ref_x.view(np.uint32)), f"x differs from {golden['commit']}"
    if name == "max_iters":
        assert st[:3].tolist() == [mi] * 3
    if zc is not None:
        assert st[zc] == 0 and not x[zc].any()
        its = [int(v) for c, v in enumerate(st[:3]) if c != zc]
        assert len(set(its)) > 1          # one channel keeps iterating after the other stopped: x-only updates
