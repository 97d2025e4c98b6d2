"""k_pcg on the device, bit for bit: iterations, residual bits and the CRC of x on three scenes equal what the k_pcg
of a9d9cb6 computed on an H100 SXM (132 SMs).  The grid has one block per SM and the grid-wide reductions add the
blocks in order, so the values hold for that SM count only; on another the test is skipped."""
import json
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMS = 132
# scene -> (loop iterations, iterations per channel, residual bits per channel, crc32 of x [R][3] float32)
EXPECTED = {
    "C1d": (80, [79, 79, 79], [952373204, 952358866, 952366236], 3788952271),
    "occ": (85, [84, 84, 84], [952491900, 952485842, 952536388], 923832063),
    "C3s": (124, [123, 123, 123], [953029812, 953018403, 953015667], 4108621762),
}

SOLVE = r"""
import importlib, json, sys, zlib
import numpy as np
sys.path.insert(0, sys.argv[1])
b2 = importlib.import_module("mvs-texturing_b200")
sc = importlib.import_module("mvs-texturing_b200.scene")
s = sc.config(sys.argv[2])
ap, ai = sc.face_adjacency(s.faces)
c = b2.Context(0)
c.set_scene(s); c.set_adjacency(ap, ai); c.set_vertex_rings(*sc.vertex_rings(s.faces, s.verts.shape[0]))
c.data_costs_run(); c.view_selection_run()
info = c.seam_run()
x = np.ascontiguousarray(c.seam_download(info)["x"], np.float32)
print(json.dumps([int(info.cg_launch_iterations), [int(v) for v in info.iterations],
                  [int(np.float32(v).view(np.uint32)) for v in info.residual], zlib.crc32(x.tobytes())]))
c.close()
"""


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _solve(name, env=None):
    r = subprocess.run([sys.executable, "-c", SOLVE, ROOT, name], capture_output=True, text=True, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-4000:]
    return tuple(json.loads(r.stdout.strip().splitlines()[-1])), r.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(EXPECTED))
def test_pcg_bit_identical_to_recorded(name):
    if _sm_count() != SMS:
        pytest.skip(f"values recorded with {SMS} SMs (one block per SM sets the reduction order)")
    got, _ = _solve(name)
    assert got == EXPECTED[name]


@pytest.mark.gpu
def test_pcg_phase_timers_do_not_change_results():
    if _sm_count() != SMS:
        pytest.skip(f"values recorded with {SMS} SMs (one block per SM sets the reduction order)")
    got, err = _solve("occ", dict(os.environ, B2TEX_SEAM_TIMING="1"))
    assert got == EXPECTED["occ"]
    assert "k_pcg: 85 iterations" in err and "spmv" in err
