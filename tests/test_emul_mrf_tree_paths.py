"""CPU half of tests/test_gpu_mrf_tree_paths.py: csrc/mrf.cu's view-selection kernels on the host emulator
(tests/cpp/emul_mrf.cpp) against the oracle, on the same synthetic grids with long-list hubs and costs on a 1/16 grid,
with 4, 8 and 16 lanes per node and the label-list cap that alloc_mrf gives those inputs under k_tree's 200 KB of
shared memory: the hubs are longer than the cap, so their trees are solved through global memory."""
import ctypes as C
import os

import numpy as np
import pytest

from test_cuda_emulation import emul  # noqa: F401  (fixture)
from test_gpu_mrf_tree_paths import tree_path_problem

pytestmark = pytest.mark.skipif(not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"),
                                reason="CUDA headers not installed")

# group: lanes per node; cap: the scratch's label-list cap.  16 warps of a block hold 16 * 32 / group lane groups, each
# with cap * 6 bytes of h row and label list plus 4 * mw bytes of bitmask and 2 * mw of prefix counts (padded to 4),
# mw = (K + 32) // 32 words; 200 KB = 204800 bytes.
CASES = {
    # 128 groups: 1600 B each; mw = 10: 40 + 20 = 60 B; (1600 - 60) / 6 = 256.7 -> 256
    "g4_hub300": dict(gen=dict(nx=32, ny=32, K=300, mean=3, hubs=(2, 2, 300, 300)), group=4, cap=256),
    # 64 groups: 3200 B each; mw = 47: 188 + 96 = 284 B; (3200 - 284) / 6 = 486 -> 480
    "g8_hub600": dict(gen=dict(nx=32, ny=32, K=1500, mean=8, hubs=(2, 2, 600, 600)), group=8, cap=480),
    # 32 groups: 6400 B each; mw = 47: 284 B; (6400 - 284) / 6 = 1019.3 -> 1008
    "g16_hub1016": dict(gen=dict(nx=32, ny=32, K=1500, mean=18, hubs=(2, 2, 1016, 1016)), group=16, cap=1008),
}


@pytest.mark.parametrize("name", list(CASES))
def test_emulated_tree_paths_match_oracle(emul, orc, name):
    case = CASES[name]
    pb = tree_path_problem(100 + sorted(CASES).index(name), **case["gen"])
    assert pb["longest"] > case["cap"]
    o = orc.view_selection(pb["ap"], pb["ai"], pb["fp"], pb["view"], pb["cost"], threads=1)
    P = dict(orc.DEFAULT_MRF)
    params = np.array([P["max_iterations"], P["rounds"], P["root_div"], P["seed"], P["window"], P["num_parts"],
                       case["group"], case["cap"], 0], np.uint32)
    F = pb["F"]
    labels = np.zeros(F, np.uint32)
    trace = np.full(P["max_iterations"] + 1, np.nan)
    stats = np.zeros(4, np.uint64)
    it = emul["emul_mrf"].emul_view_selection(C.c_uint32(F), C.c_uint32(pb["K"]), orc._p(pb["ap"]), orc._p(pb["ai"]),
                                              orc._p(pb["fp"]), orc._p(pb["view"]), orc._p(pb["cost"]), orc._p(params),
                                              C.c_float(P["ratio"]), orc._p(labels), orc._p(trace), None, orc._p(stats))
    assert it >= 0, "a kernel launch did not terminate (protocol hang)" if it == -1 else "bad parameters"
    assert it == o["iterations"]
    assert np.array_equal(trace[:it + 1], o["trace"])
    assert np.array_equal(labels, o["labels"])
    assert stats[0] > 0          # the hubs' trees went through global memory
