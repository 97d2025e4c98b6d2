"""-m gpu: gradient images of view sets the TMA kernel declines, so that k_lum_sobel computes them, against the oracle.
test_gpu_parity.py::test_gradient_images_bit_exact covers the TMA kernel (scene widths that are multiples of 16)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# (w, h, views) groups: a width that is not a multiple of 16 (3 * 317 * 239 * 5 bytes of rgb is not a multiple of 4: the
# last view's last pixel ends in a partly filled word), images smaller than one TMA box, and views of different sizes
DECLINED = {"u317x239": [(317, 239, 5)], "u120x30": [(120, 30, 4)],
            "mixed": [(317, 239, 2), (160, 120, 3), (97, 61, 2), (120, 30, 2), (2, 3, 1)]}


@pytest.mark.parametrize("name", list(DECLINED))
def test_gradient_images_of_declined_view_sets_bit_exact(b2, scene_mod, orc, name):
    """Every pixel of every gradient-magnitude image (texture_view.cpp:102-107) against the oracle; on the uniform sets
    the data costs are compared bit for bit as well, as test_data_costs_bit_exact does."""
    import torch
    from importlib import import_module
    scenes = [scene_mod.sphere_scene(6, k, w, h, displace=0.04, name=f"{name}-{w}x{h}") for w, h, k in DECLINED[name]]
    K = sum(s.num_views for s in scenes)
    views = (b2.B2View * K)()
    sizes, images = [], []
    for s in scenes:
        for v in b2.make_views(s.pos, s.viewdir, s.proj, s.w2c, s.width, s.height, s.images):
            views[len(sizes)] = v
            sizes.append((s.width, s.height))
        images += list(s.images)
    c = b2.Context(0)
    c.set_mesh(scenes[0].verts, scenes[0].faces, scenes[0].face_normals)
    c.set_views(views, K)
    info = c.data_costs_run()
    ptr, n = c.device_ptr("grad")
    total = sum(w * h for w, h in sizes)
    assert n >= total
    par = import_module("mvs-texturing_b200.sharded")
    g = torch.as_tensor(par._DevArray(ptr, total, "|u1"), device="cuda").cpu().numpy()
    d = c.data_costs_download(info.nnz, quality=True)
    c.close()
    off = 0
    for v, (w, h) in enumerate(sizes):
        ref = orc.gradient_magnitude(images[v])
        got = g[off:off + w * h].reshape(h, w)
        assert np.array_equal(got, ref), (name, v, int((got != ref).sum()))
        off += w * h
    if len(scenes) == 1:
        o = orc.data_costs(scenes[0])
        assert info.nnz == len(o["view"]) and info.nnz > 0
        assert np.array_equal(d["face_ptr"], o["face_ptr"])
        assert np.array_equal(d["view"], o["view"])
        assert np.array_equal(d["quality"].view(np.uint32), o["quality"].view(np.uint32))
        assert np.float32(info.max_quality) == np.float32(o["max_quality"])
        assert np.float32(info.percentile) == np.float32(o["percentile"])
        assert np.array_equal(d["cost"].view(np.uint32), o["cost"].view(np.uint32))
