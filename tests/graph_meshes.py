"""Meshes for the mesh-graph tests (test_emul_graph.py, test_gpu_graph.py): the non-manifold fin mesh that
tests/golden/reference_tu.npz["adjacency/fins"] records, and a seeded stress mesh with every input quirk the contract
names."""
import numpy as np


def fin_mesh(tiny):
    """`tiny` with three fins: two faces glued onto edges of face 5 and one onto an edge of face 40 (an edge shared by
    three faces), as test_ref_pinning.test_adjacency_of_non_manifold_mesh_matches_reference_tu builds it."""
    verts = np.concatenate([tiny.verts, (tiny.verts[tiny.faces[5]].mean(0) * 1.3)[None].astype(np.float32),
                            (tiny.verts[tiny.faces[40]].mean(0) * 1.3)[None].astype(np.float32)], 0)
    nv = verts.shape[0]
    fins = np.array([[tiny.faces[5][0], tiny.faces[5][1], nv - 2], [tiny.faces[5][1], tiny.faces[5][2], nv - 2],
                     [tiny.faces[40][2], tiny.faces[40][0], nv - 1]], np.uint32)
    return np.ascontiguousarray(np.concatenate([tiny.faces, fins], 0)), nv


def stress_mesh(tiny, seed=7):
    """`tiny`'s faces plus duplicate and reversed duplicate faces, faces (a,a,b) and (a,a,a), one edge shared by 40 faces,
    isolated faces and unreferenced vertices, in a shuffled order.  Returns (faces u32[F, 3], num_verts)."""
    rng = np.random.RandomState(seed)
    base = tiny.faces.astype(np.int64)
    nv = int(tiny.verts.shape[0])
    faces = [f for f in base]
    for f in rng.choice(len(base), 12, replace=False):
        faces.append(base[f].copy())
        faces.append(base[f][::-1].copy())
    a, b, c = base[3]
    faces += [np.array([a, a, b]), np.array([b, a, a]), np.array([c, c, c]), np.array([a, b, a])]
    a, b = base[10][:2]
    for k in range(40):   # a fan of 40 faces on the edge (a, b), half of them with the edge reversed
        faces.append(np.array([a, b, nv + k]) if k % 2 else np.array([nv + k, b, a]))
    nv += 40
    for _ in range(3):    # isolated triangles
        faces.append(np.array([nv, nv + 1, nv + 2]))
        nv += 3
    nv += 5               # unreferenced vertices at the end
    faces = np.array(faces, np.int64)[rng.permutation(len(faces))]
    faces = np.concatenate([faces, [[nv, nv + 2, nv + 1]]], 0)   # one more isolated face, with an unreferenced vertex
    nv += 4
    return np.ascontiguousarray(faces.astype(np.uint32)), nv


def non_manifold_edges(faces):
    """Undirected edges shared by more than two distinct faces."""
    f = faces.astype(np.int64)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]], 0)
    key = np.minimum(e[:, 0], e[:, 1]) * (int(f.max()) + 1) + np.maximum(e[:, 0], e[:, 1])
    fid = np.tile(np.arange(len(f)), 3)
    pairs = np.unique(np.stack([key, fid], 1), axis=0)
    _, cnt = np.unique(pairs[:, 0], return_counts=True)
    return int((cnt > 2).sum())
