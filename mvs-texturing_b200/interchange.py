"""On-disk interchange with a stock texrecon (SURVEY.md 8f #1, INTEGRATION.md route B).

  OUT_data_costs.spt  SparseTable<uint32,uint16,float>::save_to_file / load_from_file
                      (libs/tex/sparse_table.h:112-187): ASCII header "SPT 0.2 <cols> <rows> <nnz>\\n"
                      followed by nnz packed records (u32 col = face, u16 row = view, f32 value),
                      column major, i.e. exactly the CSR-by-face order of DataCosts.
                      Accepted by `texrecon -D` (apps/texrecon/texrecon.cpp:107-117).
  OUT_labeling.vec    vector_to_file<std::size_t> (libs/tex/util.h:104-131): raw size_t[F], no header.
                      Accepted by `texrecon -L` (texrecon.cpp:137-158).
Errors mirror the reference's util::FileException messages.
"""
from __future__ import annotations

import numpy as np

_REC = np.dtype([("col", "<u4"), ("row", "<u2"), ("val", "<f4")])  # packed: 10 bytes
assert _REC.itemsize == 10


class FileException(RuntimeError):
    pass


def save_data_costs(filename, face_ptr, view, cost, num_views):
    face_ptr = np.asarray(face_ptr, np.uint64)
    F, nnz = len(face_ptr) - 1, int(face_ptr[-1])
    rec = np.empty(nnz, _REC)
    rec["col"] = np.repeat(np.arange(F, dtype=np.uint32), np.diff(face_ptr.astype(np.int64)))
    rec["row"] = np.asarray(view, np.uint16)[:nnz]
    rec["val"] = np.asarray(cost, np.float32)[:nnz]
    with open(filename, "wb") as f:
        f.write(f"SPT 0.2 {F} {int(num_views)} {nnz}\n".encode("ascii"))
        rec.tofile(f)


def load_data_costs(filename, num_faces=None, num_views=None):
    """Returns (face_ptr u64[F+1], view u16[nnz], cost f32[nnz], num_views).  Like the reference,
    a table with different dimensions than expected is rejected (sparse_table.h:166-169)."""
    with open(filename, "rb") as f:
        header = f.readline().decode("ascii", errors="replace").split()
        if len(header) < 5 or header[0] != "SPT":
            raise FileException(f"{filename}: Not a SparseTable file!")
        if header[1] != "0.2":
            raise FileException(f"{filename}: Incompatible version of SparseTable file!")
        cols, rows, nnz = int(header[2]), int(header[3]), int(header[4])
        if (num_faces is not None and cols != num_faces) or (num_views is not None and rows != num_views):
            raise FileException(f"{filename}: SparseTable has different dimension!")
        rec = np.fromfile(f, _REC, count=nnz)
    if len(rec) != nnz:
        raise FileException(f"{filename}: truncated SparseTable file")
    col = rec["col"].astype(np.int64)
    if nnz and (np.any(np.diff(col) < 0) or col.max() >= cols):
        # set_value() order is free in the reference; DataCosts written by texrecon are column major
        order = np.argsort(col, kind="stable")
        rec, col = rec[order], col[order]
    face_ptr = np.zeros(cols + 1, np.uint64)
    np.add.at(face_ptr, col + 1, 1)
    face_ptr = np.cumsum(face_ptr).astype(np.uint64)
    return face_ptr, rec["row"].copy(), rec["val"].copy(), rows


def save_labeling(filename, labels):
    np.asarray(labels).astype("<u8").tofile(filename)  # std::size_t on LP64


def load_labeling(filename, num_faces=None, num_views=None):
    """texrecon.cpp:141-153: wrong size or label > number of views aborts."""
    lab = np.fromfile(filename, "<u8")
    if num_faces is not None and len(lab) != num_faces:
        raise FileException("Wrong labeling file for this mesh/scene combination... aborting!")
    if num_views is not None and len(lab) and lab.max() > num_views:
        raise FileException("Wrong labeling file for this mesh/scene combination... aborting!")
    return lab.astype(np.uint32)


# ------------------------------------------------------------------------------------------------------------------
# scene inputs and timings (SURVEY.md 8f #1, second half)
# ------------------------------------------------------------------------------------------------------------------
TIMING_EVENTS = ("Loading", "Calculating data costs", "Running MRF optimization", "Running global seam leveling",
                 "Calculating texture patch validity masks", "Running local seam leveling", "Building OBJ model",
                 "Saving", "Total")   # apps/texrecon/texrecon.cpp:86-211


class TimingLog:
    """OUT_timings.csv as Timer::measure / Timer::write_to_file produce it (libs/tex/timer.cpp:22-61): one row per
    event with absolute and relative clocks and milliseconds.  "Total" is relative to the start like every other
    first-of-its-kind event is not: the reference measures it against the previous event too, so do we."""

    def __init__(self, header=""):
        import time
        self._t0, self._c0 = time.perf_counter(), time.process_time()
        self.header = header
        self.events = []

    def measure(self, name, abs_ms=None, abs_clocks=None):
        import time
        if abs_ms is None:
            abs_ms = int((time.perf_counter() - self._t0) * 1000.0)
        if abs_clocks is None:
            abs_clocks = int((time.process_time() - self._c0) * 1e6)     # CLOCKS_PER_SEC = 1e6
        if self.events:
            _, pc, pm, _, _ = self.events[-1]
            rel_c, rel_m = abs_clocks - pc, abs_ms - pm
        else:
            rel_c, rel_m = abs_clocks, abs_ms
        self.events.append((name, int(abs_clocks), int(abs_ms), int(rel_c), int(rel_m)))

    def write_to_file(self, filename):
        try:
            out = open(filename, "w")
        except OSError as e:
            raise FileException(f"{filename}: {e.strerror}")
        with out:
            if self.header:
                out.write("#" + self.header + "\n")
            out.write("Event, Absolute clocks, Absolute milliseconds, Relative clocks, Relative milliseconds\n")
            for ev in self.events:
                out.write(", ".join(str(v) for v in ev) + "\n")


def load_timings(filename):
    rows = []
    with open(filename) as f:
        for line in f:
            if line.startswith("#") or line.startswith("Event,"):
                continue
            parts = [p.strip() for p in line.rstrip("\n").split(", ")]
            rows.append((parts[0],) + tuple(int(v) for v in parts[1:5]))
    return rows


def load_cam(filename, width, height):
    """MVE .cam file as generate_texture_views.cpp:118-151 reads it: line 1 = translation (3) + rotation (9, row major),
    line 2 = focal length [dist0 dist1 pixel aspect principal x y].  Returns the four quantities TextureView keeps
    (texture_view.cpp:33-39): pos, viewdir, proj (3x3, pixels), world_to_cam (4x4).  mve::CameraInfo's fill_* are
    restated [UPSTREAM-RECALL]: pos = -R^T t, viewdir = third row of R, calibration scaled by the larger image side.
    Undistortion (dist != 0, :152-162) is not applied here: pass flen and dist to Context.undistort_views after the
    images are set."""
    try:
        with open(filename) as f:
            ext = f.readline().split()
            intr = f.readline().split()
    except OSError as e:
        raise FileException(f"{filename}: {e.strerror}")
    if len(ext) != 12 or len(intr) < 1:
        raise FileException(f"Invalid CAM file: {filename}")
    t = np.array([float(v) for v in ext[:3]], np.float32)
    R = np.array([float(v) for v in ext[3:]], np.float32).reshape(3, 3)
    vals = [float(v) for v in intr] + [0.0] * 6
    flen, d0, d1 = vals[0], vals[1], vals[2]
    paspect = vals[3] if len(intr) > 3 else 1.0
    ppx = vals[4] if len(intr) > 4 else 0.5
    ppy = vals[5] if len(intr) > 5 else 0.5
    dim_aspect = float(width) / float(height)
    image_aspect = dim_aspect * paspect
    if image_aspect < 1.0:
        ax, ay = flen * height / paspect, flen * height
    else:
        ax, ay = flen * width, flen * width * paspect
    proj = np.array([[ax, 0.0, width * ppx], [0.0, ay, height * ppy], [0.0, 0.0, 1.0]], np.float32)
    w2c = np.eye(4, dtype=np.float32)
    w2c[:3, :3] = R
    w2c[:3, 3] = t
    pos = (-(R.T.astype(np.float64) @ t.astype(np.float64))).astype(np.float32)
    return dict(pos=pos, viewdir=R[2].copy(), proj=proj.ravel(), w2c=w2c.ravel(), flen=flen, dist=(d0, d1))


def save_cam(filename, w2c, flen, paspect=1.0, ppoint=(0.5, 0.5), dist=(0.0, 0.0)):
    w2c = np.asarray(w2c, np.float64).reshape(4, 4)
    with open(filename, "w") as f:
        f.write(" ".join(repr(float(v)) for v in np.r_[w2c[:3, 3], w2c[:3, :3].ravel()]) + "\n")
        f.write(f"{float(flen)!r} {float(dist[0])!r} {float(dist[1])!r} {float(paspect)!r} {float(ppoint[0])!r} {float(ppoint[1])!r}\n")


_PLY_TYPES = {"char": "i1", "uchar": "u1", "short": "i2", "ushort": "u2", "int": "i4", "uint": "u4", "float": "f4", "double": "f8",
              "int8": "i1", "uint8": "u1", "int16": "i2", "uint16": "u2", "int32": "i4", "uint32": "u4", "float32": "f4", "float64": "f8"}


def load_ply(filename):
    """Triangle mesh from a PLY file (ascii or binary little endian; texrecon reads it with mve::geom::load_ply_mesh,
    arguments.cpp:32-42).  Returns (verts f32 (Vn,3), faces u32 (F,3)); other vertex properties are skipped."""
    with open(filename, "rb") as f:
        if f.readline().strip() != b"ply":
            raise FileException(f"{filename}: not a PLY file")
        fmt, elements = None, []
        while True:
            line = f.readline()
            if not line:
                raise FileException(f"{filename}: truncated header")
            tok = line.decode("ascii", "replace").split()
            if not tok:
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                elements.append([tok[1], int(tok[2]), []])
            elif tok[0] == "property":
                elements[-1][2].append(tok[1:])
            elif tok[0] == "end_header":
                break
        if fmt not in ("ascii", "binary_little_endian"):
            raise FileException(f"{filename}: unsupported PLY format {fmt}")
        verts = faces = None
        for name, count, props in elements:
            if name == "vertex":
                names = [p[-1] for p in props]
                if fmt == "ascii":
                    rows = np.array([f.readline().split() for _ in range(count)], np.float64).reshape(count, len(props))
                    verts = rows[:, [names.index("x"), names.index("y"), names.index("z")]].astype(np.float32)
                else:
                    dt = np.dtype([(p[-1], "<" + _PLY_TYPES[p[0]]) for p in props])
                    rec = np.frombuffer(f.read(dt.itemsize * count), dt, count)
                    verts = np.stack([rec["x"], rec["y"], rec["z"]], 1).astype(np.float32)
            elif name == "face":
                lp = next(p for p in props if p[0] == "list")
                if fmt == "ascii":
                    out = []
                    for _ in range(count):
                        t = f.readline().split()
                        if int(t[0]) != 3:
                            raise FileException(f"{filename}: only triangle meshes are supported")
                        out.append([int(v) for v in t[1:4]])
                    faces = np.array(out, np.uint32).reshape(count, 3)
                else:
                    if len(props) != 1:
                        raise FileException(f"{filename}: extra face properties are not supported")
                    dt = np.dtype([("n", "<" + _PLY_TYPES[lp[1]]), ("v", "<" + _PLY_TYPES[lp[2]], 3)])
                    rec = np.frombuffer(f.read(dt.itemsize * count), dt, count)
                    if count and not (rec["n"] == 3).all():
                        raise FileException(f"{filename}: only triangle meshes are supported")
                    faces = rec["v"].astype(np.uint32)
            else:
                raise FileException(f"{filename}: unsupported element {name}")
    if verts is None or faces is None:
        raise FileException(f"{filename}: vertex or face element missing")
    return np.ascontiguousarray(verts), np.ascontiguousarray(faces)


def save_ply(filename, verts, faces, binary=True):
    verts, faces = np.asarray(verts, np.float32), np.asarray(faces, np.uint32)
    with open(filename, "wb") as f:
        f.write(("ply\nformat %s 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
                 "element face %d\nproperty list uchar int vertex_indices\nend_header\n"
                 % ("binary_little_endian" if binary else "ascii", len(verts), len(faces))).encode())
        if binary:
            f.write(verts.astype("<f4").tobytes())
            rec = np.zeros(len(faces), np.dtype([("n", "u1"), ("v", "<i4", 3)]))
            rec["n"], rec["v"] = 3, faces
            f.write(rec.tobytes())
        else:
            for v in verts:
                f.write(("%r %r %r\n" % tuple(float(x) for x in v)).encode())
            for t in faces:
                f.write(("3 %d %d %d\n" % tuple(int(x) for x in t)).encode())
