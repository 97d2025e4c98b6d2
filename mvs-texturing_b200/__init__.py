"""mvs-texturing_b200 -- CUDA hot path of nmoehrle/mvs-texturing for the H100.

Host-side binding of include/b2tex.h (libb2tex.so, hand-written sm_90a CUDA).  The functions at
the bottom mirror the reference's operator interface for the path (libs/tex/texturing.h:66-106):

    calculate_data_costs(mesh, texture_views, settings) -> DataCosts      (texturing.h:66-69)
    view_selection(data_costs, graph, settings)          -> labels         (texturing.h:79-80)
    global_seam_leveling(graph_labels, mesh, rings, texture_views) -> adjust values (texturing.h:97-101)

There is no CPU fallback: importing works anywhere (the library is only dlopen'ed on first use),
but every call raises if libb2tex.so is missing or no CUDA device is present.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb2tex.so")

EXPORTS = [
    "b2tex_create", "b2tex_destroy", "b2tex_last_error", "b2tex_free", "b2tex_device_synchronize",
    "b2tex_stream", "b2tex_launch_count", "b2tex_profile", "b2tex_profile_report",
    "b2tex_default_mrf_params", "b2tex_texrecon_mrf_params", "b2tex_set_mesh", "b2tex_set_views", "b2tex_set_adjacency",
    "b2tex_set_vertex_rings", "b2tex_set_data_costs", "b2tex_set_labels", "b2tex_set_face_range", "b2tex_undistort_views",
    "b2tex_data_costs_run", "b2tex_data_costs_qualities", "b2tex_data_costs_histogram",
    "b2tex_data_costs_normalize", "b2tex_data_costs_download", "b2tex_view_selection_run", "b2tex_view_selection_prepare",
    "b2tex_labels_download", "b2tex_mrf_init", "b2tex_mrf_iterate", "b2tex_mrf_energy", "b2tex_mrf_sample_forest",
    "b2tex_seam_run", "b2tex_seam_download", "b2tex_seam_matrix_download", "b2tex_device_ptr",
    "b2tex_texture_patches_run", "b2tex_texture_patches_download", "b2tex_local_seam_leveling_run", "b2tex_seam_assemble", "b2tex_seam_mg_export", "b2tex_seam_mg_import",
    "b2tex_seam_mg_solve", "b2tex_mrf_mg_export", "b2tex_mrf_mg_import", "b2tex_peer_block", "b2tex_peer_attach",
    "b2tex_calculate_data_costs", "b2tex_calculate_data_costs_into", "b2tex_postprocess_face_infos", "b2tex_view_selection",
    "b2tex_global_seam_leveling", "b2tex_texture_hot_path", "b2tex_seam_leveling_patches", "b2tex_release_cached_contexts",
    "b2tex_build_mesh_graph", "b2tex_mesh_graph_download", "b2tex_prepare_mesh", "b2tex_prepared_mesh_download",
]


class B2View(C.Structure):
    _fields_ = [("pos", C.c_float * 3), ("viewdir", C.c_float * 3), ("proj", C.c_float * 9),
                ("w2c", C.c_float * 16), ("width", C.c_int32), ("height", C.c_int32),
                ("rgb", C.c_void_p)]


class B2Distortion(C.Structure):
    _fields_ = [("flen", C.c_float), ("dist", C.c_float * 2)]


class B2Settings(C.Structure):
    _fields_ = [("data_term", C.c_int32), ("outlier_removal", C.c_int32),
                ("geometric_visibility_test", C.c_int32)]


class B2DcInfo(C.Structure):
    _fields_ = [("nnz", C.c_uint64), ("candidates", C.c_uint64), ("rays", C.c_uint64),
                ("max_quality", C.c_float), ("percentile", C.c_float)]


class B2MrfParams(C.Structure):
    _fields_ = [("max_iterations", C.c_uint32), ("rounds", C.c_uint32), ("root_div", C.c_uint32),
                ("seed", C.c_uint32), ("window", C.c_uint32), ("ratio", C.c_float),
                ("num_parts", C.c_uint32), ("num_views", C.c_uint32), ("use_multilevel", C.c_uint32),
                ("use_spanning_tree", C.c_uint32), ("spanning_tree_multilevel_after_n_iterations", C.c_uint32)]


class B2MrfInfo(C.Structure):
    _fields_ = [("iterations", C.c_uint32), ("energy_initial", C.c_double),
                ("energy_final", C.c_double), ("unseen", C.c_uint64), ("sweep_bytes", C.c_uint64),
                ("multilevel_passes", C.c_uint32), ("coarse_nodes", C.c_uint32),
                ("spanning_tree_iterations", C.c_uint32), ("spanning_tree_rejected", C.c_uint32),
                ("tree_group", C.c_uint32), ("tree_cap", C.c_uint32), ("label_mask_words", C.c_uint32),
                ("global_trees", C.c_uint32), ("multilevel_steps", C.c_uint32),
                ("multilevel_steps_rejected", C.c_uint32)]


class B2PatchInfo(C.Structure):
    _fields_ = [("num_patches", C.c_uint32), ("num_faces", C.c_uint32), ("num_pixels", C.c_uint64)]


class B2LocalSeamInfo(C.Structure):
    _fields_ = [("num_seam_edges", C.c_uint32), ("num_edge_samples", C.c_uint32), ("num_vertices", C.c_uint32),
                ("num_unknowns", C.c_uint32), ("iterations", C.c_uint32 * 3), ("residual", C.c_float * 3)]


class B2SeamInfo(C.Structure):
    _fields_ = [("num_rows", C.c_uint32), ("num_a_rows", C.c_uint32), ("num_gamma_rows", C.c_uint32),
                ("nnz_full", C.c_uint64), ("iterations", C.c_uint32 * 3), ("residual", C.c_float * 3),
                ("cg_launch_iterations", C.c_uint32), ("cg_ms", C.c_float)]


class B2GraphInfo(C.Structure):
    _fields_ = [("num_adjacency", C.c_uint32), ("num_vertex_faces", C.c_uint32), ("num_vertex_neighbours", C.c_uint32),
                ("max_face_degree", C.c_uint32), ("num_non_manifold_edges", C.c_uint32)]


class B2MeshPrepInfo(C.Structure):
    _fields_ = [("num_faces_in", C.c_uint32), ("num_faces", C.c_uint32), ("num_redundant", C.c_uint32),
                ("num_zero_normals", C.c_uint32), ("graph", B2GraphInfo)]


class B2TexError(RuntimeError):
    def __init__(self, rc, msg):
        super().__init__(f"b2tex error {rc}: {msg}")
        self.rc = rc


_lib = None


def lib():
    """dlopen libb2tex.so; fails loudly if the CUDA extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`"
                              " -- the product path has no CPU fallback")
        L = C.CDLL(LIB_PATH)
        L.b2tex_last_error.restype = C.c_char_p
        L.b2tex_device_ptr.restype = C.c_uint64
        L.b2tex_stream.restype = C.c_uint64
        L.b2tex_launch_count.restype = C.c_uint64
        L.b2tex_peer_block.restype = C.c_uint64
        _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        raise B2TexError(rc, lib().b2tex_last_error().decode(errors="replace"))


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _c(a, dt):
    return np.ascontiguousarray(a, dtype=dt)


def make_views(pos, viewdir, proj, w2c, width, height, images):
    """Pack camera arrays + (K,H,W,3) u8 images into an array of b2tex_view."""
    K = len(pos)
    arr = (B2View * K)()
    for k in range(K):
        arr[k].pos[:] = np.asarray(pos[k], np.float32).tolist()
        arr[k].viewdir[:] = np.asarray(viewdir[k], np.float32).tolist()
        arr[k].proj[:] = np.asarray(proj[k], np.float32).ravel().tolist()
        arr[k].w2c[:] = np.asarray(w2c[k], np.float32).ravel().tolist()
        arr[k].width = int(width)
        arr[k].height = int(height)
        arr[k].rgb = images[k].ctypes.data
    return arr


def mrf_params(**kw) -> B2MrfParams:
    p = B2MrfParams()
    lib().b2tex_default_mrf_params(C.byref(p))
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def texrecon_mrf_params(**kw) -> B2MrfParams:
    """mrf_params with mapMAP's control as texrecon sets it (b2tex_texrecon_mrf_params): use_spanning_tree = 1,
    use_multilevel = 1, spanning_tree_multilevel_after_n_iterations = 5; `kw` on top."""
    p = B2MrfParams()
    lib().b2tex_texrecon_mrf_params(C.byref(p))
    for k, v in kw.items():
        setattr(p, k, v)
    return p


class Context:
    """Resident API: upload once, run stages on the device (b2tex_ctx)."""

    def __init__(self, device: int = 0):
        self._h = C.c_void_p()
        _check(lib().b2tex_create(C.c_int(device), C.byref(self._h)))
        self.F = self.Vn = self.K = 0
        self._keep = []

    def close(self):
        if self._h:
            lib().b2tex_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- uploads ----
    def set_mesh(self, verts, faces, face_normals):
        v, f, n = _c(verts, np.float32), _c(faces, np.uint32), _c(face_normals, np.float32)
        self.Vn, self.F = v.shape[0], f.shape[0]
        _check(lib().b2tex_set_mesh(self._h, _p(v), C.c_uint32(self.Vn), _p(f), _p(n), C.c_uint32(self.F)))

    def set_views(self, views, K):
        self.K = K
        _check(lib().b2tex_set_views(self._h, views, C.c_uint32(K)))

    def set_scene(self, scene, images=None):
        self.set_mesh(scene.verts, scene.faces, scene.face_normals)
        imgs = scene.images if images is None else images
        self.set_views(make_views(scene.pos, scene.viewdir, scene.proj, scene.w2c, scene.width,
                                  scene.height, imgs), scene.num_views)

    def undistort_views(self, flen, dist):
        """Undistort the resident images in place, as the reference does for .cam views (b2tex_undistort_views).
        flen[K]: focal lengths normalised by the larger image side; dist[K, 2]: .cam radial coefficients.  A view with
        dist[v, 0] == 0 is left as it is; dist[v, 1] != 0 selects the Bundler k2 k4 model, otherwise VisualSFM's.
        Call after set_views / set_scene and before the stages."""
        flen = np.asarray(flen, np.float32).reshape(-1)
        dist = np.asarray(dist, np.float32).reshape(-1, 2)
        if len(flen) != len(dist):
            raise ValueError(f"undistort_views: {len(flen)} focal lengths for {len(dist)} distortions")
        d = (B2Distortion * max(len(flen), 1))()
        for v in range(len(flen)):
            d[v].flen = float(flen[v])
            d[v].dist[:] = dist[v].tolist()
        _check(lib().b2tex_undistort_views(self._h, d, C.c_uint32(len(flen))))

    def set_adjacency(self, adj_ptr, adj_idx):
        _check(lib().b2tex_set_adjacency(self._h, _p(_c(adj_ptr, np.uint32)), _p(_c(adj_idx, np.uint32))))

    def set_vertex_rings(self, vf_ptr, vf_idx, vv_ptr, vv_idx):
        _check(lib().b2tex_set_vertex_rings(self._h, _p(_c(vf_ptr, np.uint32)), _p(_c(vf_idx, np.uint32)),
                                            _p(_c(vv_ptr, np.uint32)), _p(_c(vv_idx, np.uint32))))

    def build_mesh_graph(self) -> B2GraphInfo:
        """Derive the face adjacency and the vertex rings from the resident mesh on the device (b2tex_build_mesh_graph):
        afterwards the context is as after set_adjacency / set_vertex_rings with scene.face_adjacency /
        scene.vertex_rings.  Call after set_mesh / set_scene."""
        info = B2GraphInfo()
        _check(lib().b2tex_build_mesh_graph(self._h, C.byref(info)))
        return info

    def mesh_graph_download(self, info: B2GraphInfo):
        """the resident graph as dict(adj_ptr, adj_idx, vf_ptr, vf_idx, vv_ptr, vv_idx), sized from build_mesh_graph's info"""
        out = dict(adj_ptr=np.zeros(self.F + 1, np.uint32), adj_idx=np.zeros(info.num_adjacency, np.uint32),
                   vf_ptr=np.zeros(self.Vn + 1, np.uint32), vf_idx=np.zeros(info.num_vertex_faces, np.uint32),
                   vv_ptr=np.zeros(self.Vn + 1, np.uint32), vv_idx=np.zeros(info.num_vertex_neighbours, np.uint32))
        _check(lib().b2tex_mesh_graph_download(self._h, *(_p(out[k]) for k in
                                                         ("adj_ptr", "adj_idx", "vf_ptr", "vf_idx", "vv_ptr", "vv_idx"))))
        return out

    def prepare_mesh(self, verts, faces) -> B2MeshPrepInfo:
        """tex::prepare_mesh on the raw mesh (b2tex_prepare_mesh), e.g. the arrays of interchange.load_ply: drops the
        redundant faces (face i goes when a face j > i has all its vertices among those of i), computes the face normals of
        the kept faces, the mesh graph and the vertex normals.  Afterwards the context is as after set_mesh(verts, kept
        faces, scene.face_normals of them) + build_mesh_graph; self.F is the kept count."""
        v, f = _c(verts, np.float32), _c(faces, np.uint32)
        info = B2MeshPrepInfo()
        self.F = 0
        _check(lib().b2tex_prepare_mesh(self._h, _p(v), C.c_uint32(v.shape[0]), _p(f), C.c_uint32(f.shape[0]),
                                        C.byref(info)))
        self.Vn, self.F = v.shape[0], int(info.num_faces)
        return info

    def prepared_mesh_download(self, info: B2MeshPrepInfo):
        """dict(faces u32[F', 3], face_normals f32[F', 3], vertex_normals f32[Vn, 3], kept u32[F']): kept[i] is the input
        id of face i, which maps per-face results back to the file's face ids"""
        F = int(info.num_faces)
        out = dict(faces=np.zeros((F, 3), np.uint32), face_normals=np.zeros((F, 3), np.float32),
                   vertex_normals=np.zeros((self.Vn, 3), np.float32), kept=np.zeros(F, np.uint32))
        _check(lib().b2tex_prepared_mesh_download(self._h, *(_p(out[k]) for k in
                                                            ("faces", "face_normals", "vertex_normals", "kept"))))
        return out

    def set_num_faces(self, F):
        """For view selection without a mesh (the reference's view_selection never sees one)."""
        raise NotImplementedError("use the one-shot view_selection() for mesh-less calls")

    def set_data_costs(self, face_ptr, view, cost):
        _check(lib().b2tex_set_data_costs(self._h, _p(_c(face_ptr, np.uint64)), _p(_c(view, np.uint16)),
                                          _p(_c(cost, np.float32))))

    def set_labels(self, labels):
        _check(lib().b2tex_set_labels(self._h, _p(_c(labels, np.uint32))))

    def set_face_range(self, begin, end):
        _check(lib().b2tex_set_face_range(self._h, C.c_uint32(begin), C.c_uint32(end)))

    @staticmethod
    def launch_count() -> int:
        """kernels of libb2tex.so launched by this process so far"""
        return int(lib().b2tex_launch_count())

    def synchronize(self):
        _check(lib().b2tex_device_synchronize(self._h))

    def stream(self) -> int:
        return int(lib().b2tex_stream(self._h))

    def profile(self, enable=True):
        _check(lib().b2tex_profile(self._h, C.c_int(1 if enable else 0)))

    def profile_report(self):
        """list of (name, ms, algorithmic_bytes) per recorded launch group since profile(True)"""
        buf = C.create_string_buffer(1 << 20)
        lib().b2tex_profile_report(self._h, buf, C.c_uint64(len(buf)))
        out = []
        for line in buf.value.decode().splitlines():
            name, ms, by = line.rsplit(" ", 2)
            out.append((name, float(ms), float(by)))
        return out

    # ---- stages ----
    def data_costs_run(self, data_term=1, visibility=True, outlier_removal=0):
        st = B2Settings(data_term, outlier_removal, 1 if visibility else 0)
        info = B2DcInfo()
        _check(lib().b2tex_data_costs_run(self._h, C.byref(st), C.byref(info)))
        return info

    def data_costs_qualities(self, data_term=1, visibility=True, outlier_removal=0):
        st = B2Settings(data_term, outlier_removal, 1 if visibility else 0)
        info = B2DcInfo()
        _check(lib().b2tex_data_costs_qualities(self._h, C.byref(st), C.byref(info)))
        return info

    def data_costs_histogram(self, gmax):
        bins = np.zeros(10000, np.uint32)
        _check(lib().b2tex_data_costs_histogram(self._h, C.c_float(gmax), _p(bins), C.c_int(1)))
        return bins

    def data_costs_histogram_device(self, gmax):
        """histogram stays on the device (buffer "hist") so that NCCL can all-reduce it in place"""
        _check(lib().b2tex_data_costs_histogram(self._h, C.c_float(gmax), None, C.c_int(0)))

    def data_costs_normalize(self, gmax, bins):
        info = B2DcInfo()
        _check(lib().b2tex_data_costs_normalize(self._h, C.c_float(gmax), _p(_c(bins, np.uint32)), C.byref(info)))
        return info

    def data_costs_download(self, nnz, quality=False):
        face_ptr = np.zeros(self.F + 1, np.uint64)
        view = np.zeros(nnz, np.uint16)
        cost = np.zeros(nnz, np.float32)
        q = np.zeros(nnz, np.float32) if quality else None
        _check(lib().b2tex_data_costs_download(self._h, _p(face_ptr), _p(view), _p(cost), _p(q)))
        return dict(face_ptr=face_ptr, view=view, cost=cost, quality=q)

    def view_selection_prepare(self, **kw):
        p = mrf_params(**kw)
        _check(lib().b2tex_view_selection_prepare(self._h, C.byref(p)))

    def view_selection_run(self, **kw):
        p = mrf_params(**kw)
        info = B2MrfInfo()
        trace = np.full(p.max_iterations + 1, np.nan)
        _check(lib().b2tex_view_selection_run(self._h, C.byref(p), C.byref(info), _p(trace)))
        return info, trace[:info.iterations + 1].copy()

    # multi-GPU view selection (csrc/mrf.cu): peer-visible label block; handles are exchanged by the caller
    def mrf_mg_export(self, rank, num_ranks) -> bytes:
        h = C.create_string_buffer(64)
        _check(lib().b2tex_mrf_mg_export(self._h, C.c_uint32(rank), C.c_uint32(num_ranks), h))
        return h.raw

    def mrf_mg_import(self, peer_rank, handle: bytes):
        _check(lib().b2tex_mrf_mg_import(self._h, C.c_uint32(peer_rank), C.c_char_p(handle)))

    def peer_block(self, which) -> int:
        """raw device pointer of the own peer block (0 = view selection, 1 = seam solve) for same-process peers"""
        return int(lib().b2tex_peer_block(self._h, C.c_int(which)))

    def peer_attach(self, which, peer_rank, ptr):
        _check(lib().b2tex_peer_attach(self._h, C.c_int(which), C.c_uint32(peer_rank), C.c_uint64(ptr)))

    def mrf_init(self, **kw):
        p = mrf_params(**kw)
        e = C.c_int64()
        _check(lib().b2tex_mrf_init(self._h, C.byref(p), C.byref(e)))
        return e.value

    def mrf_iterate(self, t):
        e = C.c_int64()
        _check(lib().b2tex_mrf_iterate(self._h, C.c_uint32(t), C.byref(e)))
        return e.value

    def mrf_energy(self):
        e = C.c_int64()
        _check(lib().b2tex_mrf_energy(self._h, C.byref(e)))
        return e.value

    def mrf_sample_forest(self, iteration, **kw):
        p = mrf_params(**kw)
        level = np.zeros(self.F, np.uint32)
        _check(lib().b2tex_mrf_sample_forest(self._h, C.byref(p), C.c_uint32(iteration), _p(level)))
        return level

    def labels_download(self):
        labels = np.zeros(self.F, np.uint32)
        _check(lib().b2tex_labels_download(self._h, _p(labels)))
        return labels

    def seam_run(self):
        info = B2SeamInfo()
        _check(lib().b2tex_seam_run(self._h, C.byref(info)))
        return info

    # multi-GPU seam solve (csrc/seam_mg.cu): assemble, exchange the IPC handles of the peer blocks, solve
    def seam_assemble(self):
        info = B2SeamInfo()
        _check(lib().b2tex_seam_assemble(self._h, C.byref(info)))
        return info

    def seam_mg_export(self, rank, num_ranks) -> bytes:
        h = C.create_string_buffer(64)
        _check(lib().b2tex_seam_mg_export(self._h, C.c_uint32(rank), C.c_uint32(num_ranks), h))
        return h.raw

    def seam_mg_import(self, peer_rank, handle: bytes):
        _check(lib().b2tex_seam_mg_import(self._h, C.c_uint32(peer_rank), C.c_char_p(handle)))

    def seam_mg_solve(self, info):
        _check(lib().b2tex_seam_mg_solve(self._h, C.byref(info)))
        return info

    def seam_download(self, info, rhs=False):
        R = int(info.num_rows)
        row_ptr = np.zeros(self.Vn + 1, np.uint32)
        row_label = np.zeros(R, np.uint32)
        x = np.zeros((R, 3), np.float32)
        r = np.zeros((R, 3), np.float32) if rhs else None
        _check(lib().b2tex_seam_download(self._h, _p(row_ptr), _p(row_label), _p(x), _p(r)))
        return dict(row_ptr=row_ptr, row_label=row_label, x=x, rhs=r)

    def texture_patches_run(self, apply_adjust=True):
        """tex::generate_texture_patches (seen faces) + TexturePatch::adjust_colors per patch"""
        info = B2PatchInfo()
        _check(lib().b2tex_texture_patches_run(self._h, C.c_int(1 if apply_adjust else 0), C.byref(info)))
        return info

    def local_seam_leveling_run(self):
        """tex::local_seam_leveling on the resident texture patches"""
        info = B2LocalSeamInfo()
        _check(lib().b2tex_local_seam_leveling_run(self._h, C.byref(info)))
        return info

    def texture_patches_download(self, info):
        """list of dicts: label, min_x, min_y, faces, texcoords (3n x 2), image (h x w x 3), validity, blending"""
        n, T, P = int(info.num_patches), int(info.num_faces), int(info.num_pixels)
        desc = np.zeros((max(n, 1), 8), np.int32)
        faces = np.zeros(max(T, 1), np.uint32)
        tex = np.zeros((max(T, 1) * 3, 2), np.float32)
        img = np.zeros((max(P, 1), 3), np.float32)
        val = np.zeros(max(P, 1), np.uint8)
        bl = np.zeros(max(P, 1), np.uint8)
        _check(lib().b2tex_texture_patches_download(self._h, _p(desc), _p(faces), _p(tex), _p(img), _p(val), _p(bl)))
        out, off = [], 0
        for q in range(n):
            label, mx, my, w, h, first, nf, _ = (int(v) for v in desc[q])
            out.append(dict(label=label, min_x=mx, min_y=my, faces=faces[first:first + nf].tolist(),
                            texcoords=tex[3 * first:3 * (first + nf)].copy(), image=img[off:off + w * h].reshape(h, w, 3).copy(),
                            validity=val[off:off + w * h].reshape(h, w).copy(), blending=bl[off:off + w * h].reshape(h, w).copy()))
            off += w * h
        return out

    def seam_matrix(self, info):
        R, nz = int(info.num_rows), int(info.nnz_full)
        cp, cc, cv = np.zeros(R + 1, np.uint32), np.zeros(nz, np.uint32), np.zeros(nz, np.float32)
        _check(lib().b2tex_seam_matrix_download(self._h, _p(cp), _p(cc), _p(cv)))
        return cp, cc, cv

    def device_ptr(self, name):
        n = C.c_uint64()
        p = lib().b2tex_device_ptr(self._h, name.encode(), C.byref(n))
        return int(p), int(n.value)


# ------------------------------------------------------------------------------------------------
# Reference-shaped operators (one-shot, host buffers in and out) -- libs/tex/texturing.h
# ------------------------------------------------------------------------------------------------
class Settings:
    """tex::Settings (libs/tex/settings.h:82-94), the fields this path reads."""
    DATA_TERM_AREA, DATA_TERM_GMI = 0, 1
    OUTLIER_REMOVAL_NONE, OUTLIER_REMOVAL_GAUSS_DAMPING, OUTLIER_REMOVAL_GAUSS_CLAMPING = 0, 1, 2

    def __init__(self, data_term=1, outlier_removal=0, geometric_visibility_test=True):
        self.data_term = data_term
        self.outlier_removal = outlier_removal
        self.geometric_visibility_test = geometric_visibility_test


class DataCosts:
    """tex::DataCosts = SparseTable<u32 face, u16 view, float> (texturing.h:36) as CSR by face."""

    def __init__(self, num_faces, num_views, face_ptr, view, cost):
        self.cols_, self.rows_ = num_faces, num_views
        self.face_ptr, self.view, self.cost = face_ptr, view, cost

    def cols(self):
        return self.cols_

    def rows(self):
        return self.rows_

    def col(self, i):
        a, b = int(self.face_ptr[i]), int(self.face_ptr[i + 1])
        return list(zip(self.view[a:b].tolist(), self.cost[a:b].tolist()))

    def get_nnz(self):
        return int(self.face_ptr[-1])


def _grab(ptr, ctype, n):
    a = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), (max(int(n), 1),))[:int(n)].copy()
    lib().b2tex_free(ptr)
    return a


def calculate_data_costs(scene, settings: Settings | None = None, out=None) -> DataCosts:
    """tex::calculate_data_costs (calculate_data_costs.cpp:308-323) through b2tex_calculate_data_costs.
    `out` = (face_ptr u64[F+1], view u16[cap], cost f32[cap]) caller-owned (pinned) buffers: the
    result is written in place (b2tex_calculate_data_costs_into), no allocation or extra copy."""
    st = settings or Settings()
    if out is not None:
        views = make_views(scene.pos, scene.viewdir, scene.proj, scene.w2c, scene.width, scene.height, scene.images)
        s = B2Settings(st.data_term, st.outlier_removal, 1 if st.geometric_visibility_test else 0)
        info = B2DcInfo()
        v, f, n = _c(scene.verts, np.float32), _c(scene.faces, np.uint32), _c(scene.face_normals, np.float32)
        fp, vw, cs = out
        _check(lib().b2tex_calculate_data_costs_into(_p(v), C.c_uint32(v.shape[0]), _p(f), _p(n), C.c_uint32(f.shape[0]),
                                                     views, C.c_uint32(scene.num_views), C.byref(s), _p(fp), _p(vw),
                                                     _p(cs), C.c_uint64(len(vw)), C.byref(info)))
        dc = DataCosts(f.shape[0], scene.num_views, fp, vw[:info.nnz], cs[:info.nnz])
        dc.info = info
        return dc
    if scene.num_views > 65535:
        raise RuntimeError("Exeeded maximal number of views")
    views = make_views(scene.pos, scene.viewdir, scene.proj, scene.w2c, scene.width, scene.height, scene.images)
    s = B2Settings(st.data_term, st.outlier_removal, 1 if st.geometric_visibility_test else 0)
    fp, vw, cs = C.c_void_p(), C.c_void_p(), C.c_void_p()
    info = B2DcInfo()
    v, f, n = _c(scene.verts, np.float32), _c(scene.faces, np.uint32), _c(scene.face_normals, np.float32)
    _check(lib().b2tex_calculate_data_costs(_p(v), C.c_uint32(v.shape[0]), _p(f), _p(n), C.c_uint32(f.shape[0]),
                                            views, C.c_uint32(scene.num_views), C.byref(s), C.byref(fp),
                                            C.byref(vw), C.byref(cs), C.byref(info)))
    F = f.shape[0]
    dc = DataCosts(F, scene.num_views, _grab(fp, C.c_uint64, F + 1), _grab(vw, C.c_uint16, info.nnz),
                   _grab(cs, C.c_float, info.nnz))
    dc.info = info
    return dc


def view_selection(data_costs: DataCosts, adj_ptr, adj_idx, settings: Settings | None = None, **mrf_kw):
    """tex::view_selection (view_selection.cpp:18-133): returns (labels[F], info)."""
    p = mrf_params(num_views=data_costs.rows(), **mrf_kw)
    F = data_costs.cols()
    labels = np.zeros(F, np.uint32)
    info = B2MrfInfo()
    _check(lib().b2tex_view_selection(C.c_uint32(F), _p(_c(adj_ptr, np.uint32)), _p(_c(adj_idx, np.uint32)),
                                      _p(_c(data_costs.face_ptr, np.uint64)), _p(_c(data_costs.view, np.uint16)),
                                      _p(_c(data_costs.cost, np.float32)), C.byref(p), _p(labels), C.byref(info)))
    return labels, info


def global_seam_leveling(scene, rings, labels):
    """tex::global_seam_leveling up to adjust_values (global_seam_leveling.cpp:140-291).
    rings=None: the vertex rings are derived from the mesh on the device."""
    views = make_views(scene.pos, scene.viewdir, scene.proj, scene.w2c, scene.width, scene.height, scene.images)
    vf_ptr, vf_idx, vv_ptr, vv_idx = [None] * 4 if rings is None else [None if a is None else _c(a, np.uint32) for a in rings]
    v, f = _c(scene.verts, np.float32), _c(scene.faces, np.uint32)
    Vn = v.shape[0]
    row_ptr = np.zeros(Vn + 1, np.uint32)
    rl, x = C.c_void_p(), C.c_void_p()
    info = B2SeamInfo()
    _check(lib().b2tex_global_seam_leveling(_p(v), C.c_uint32(Vn), _p(f), C.c_uint32(f.shape[0]), _p(vf_ptr),
                                            _p(vf_idx), _p(vv_ptr), _p(vv_idx), _p(_c(labels, np.uint32)), views,
                                            C.c_uint32(scene.num_views), _p(row_ptr), C.byref(rl), C.byref(x),
                                            C.byref(info)))
    R = int(info.num_rows)
    return dict(row_ptr=row_ptr, row_label=_grab(rl, C.c_uint32, R),
                x=_grab(x, C.c_float, 3 * R).reshape(R, 3), info=info)


def texture_hot_path(scene, adj, rings, settings: Settings | None = None, **mrf_kw):
    """calculate_data_costs -> view_selection -> global_seam_leveling on ONE upload
    (b2tex_texture_hot_path): host buffers in, labels + adjust values out, DataCosts stay on the device.
    adj=None, rings=None: the face adjacency and the vertex rings are derived from the mesh on the device (both or
    neither: a mix raises B2TexError)."""
    st = settings or Settings()
    views = make_views(scene.pos, scene.viewdir, scene.proj, scene.w2c, scene.width, scene.height, scene.images)
    s = B2Settings(st.data_term, st.outlier_removal, 1 if st.geometric_visibility_test else 0)
    p = mrf_params(**mrf_kw)
    v, f, n = _c(scene.verts, np.float32), _c(scene.faces, np.uint32), _c(scene.face_normals, np.float32)
    ap, ai = (None, None) if adj is None else (_c(adj[0], np.uint32), _c(adj[1], np.uint32))
    vf_ptr, vf_idx, vv_ptr, vv_idx = [None] * 4 if rings is None else [_c(a, np.uint32) for a in rings]
    Vn, F = v.shape[0], f.shape[0]
    labels = np.zeros(F, np.uint32)
    row_ptr = np.zeros(Vn + 1, np.uint32)
    rl, x = C.c_void_p(), C.c_void_p()
    dci, mi, si = B2DcInfo(), B2MrfInfo(), B2SeamInfo()
    _check(lib().b2tex_texture_hot_path(_p(v), C.c_uint32(Vn), _p(f), _p(n), C.c_uint32(F), views,
                                        C.c_uint32(scene.num_views), _p(ap), _p(ai), _p(vf_ptr), _p(vf_idx),
                                        _p(vv_ptr), _p(vv_idx), C.byref(s), C.byref(p), _p(labels), _p(row_ptr),
                                        C.byref(rl), C.byref(x), C.byref(dci), C.byref(mi), C.byref(si)))
    R = int(si.num_rows)
    return dict(labels=labels, row_ptr=row_ptr, row_label=_grab(rl, C.c_uint32, R),
                x=_grab(x, C.c_float, 3 * R).reshape(R, 3), dc_info=dci, mrf_info=mi, seam_info=si)
