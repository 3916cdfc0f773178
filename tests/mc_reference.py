"""Numpy twin of the marching-cubes kernels (csrc/mcubes.cu): same case table, same output order, float32 arithmetic.

Vertices are ordered by (grid point linear index, axis) of their edge, faces by (cube linear index, table order).
A vertex is ``lower + t`` along its edge's axis with ``t = (thr - v_lower) / (v_upper - v_lower)``, every step
rounded to float32 as the kernel's ``__fsub_rn`` / ``__fdiv_rn`` / ``__fadd_rn`` do.
"""
import numpy as np

from neddf_b200 import mc_table as T

TRI_COUNT = np.array([len(t) for t in T.TABLE], np.int64)
EDGE_MASK = np.array(T.EDGE_MASK, np.int64)
TRI_EDGES = np.full((256, 3 * T.MAX_TRIS), -1, np.int64)
for _c, _tris in enumerate(T.TABLE):
    _flat = [e for t in _tris for e in t]
    TRI_EDGES[_c, :len(_flat)] = _flat


def classify(vol: np.ndarray, thr: float) -> np.ndarray:
    """Case byte of every cube [n0-1, n1-1, n2-1] (0 for a cube with a non-finite corner)."""
    v = np.asarray(vol, np.float32)
    n0, n1, n2 = v.shape
    thr = np.float32(thr)
    case = np.zeros((n0 - 1, n1 - 1, n2 - 1), np.int64)
    finite = np.ones(case.shape, bool)
    for b, (di, dj, dk) in enumerate(T.CORNERS):
        c = v[di:di + n0 - 1, dj:dj + n1 - 1, dk:dk + n2 - 1]
        finite &= np.isfinite(c)
        case |= (c < thr).astype(np.int64) << b
    case[~finite] = 0
    return case


def marching_cubes(vol: np.ndarray, thr: float):
    """(vertices [V,3] float32, faces [F,3] int64) in index space, as neddf_b200.mesh.marching_cubes returns them."""
    v = np.ascontiguousarray(vol, np.float32)
    n0, n1, n2 = v.shape
    thr32 = np.float32(thr)
    case = classify(v, thr)
    emit = TRI_COUNT[case] > 0
    flags = np.zeros((n0, n1, n2, 3), bool)
    for e, (b, axis) in enumerate(T.EDGES):
        di, dj, dk = T.CORNERS[b]
        used = emit & (((EDGE_MASK[case] >> e) & 1) == 1)
        flags[di:di + n0 - 1, dj:dj + n1 - 1, dk:dk + n2 - 1, axis] |= used
    flat = flags.reshape(-1)
    ids = np.cumsum(flat, dtype=np.int64) - flat
    slots = np.nonzero(flat)[0]
    g, axis = slots // 3, slots % 3
    step = np.array([n1 * n2, n2, 1], np.int64)[axis]
    vf = v.reshape(-1)
    v0, v1 = vf[g], vf[g + step]
    with np.errstate(divide="ignore", invalid="ignore"):
        t = (thr32 - v0) / (v1 - v0)
    verts = np.stack(np.unravel_index(g, (n0, n1, n2)), 1).astype(np.float32)
    rows = np.arange(len(slots))
    verts[rows, axis] = verts[rows, axis] + t
    # faces: emitting cubes in linear order, each cube's triangles in table order
    cubes = np.nonzero(emit.reshape(-1))[0]
    ci, cj, ck = np.unravel_index(cubes, case.shape)
    base = (ci * n1 + cj) * n2 + ck
    edges = TRI_EDGES[case.reshape(-1)[cubes]]                       # [n, 15], -1 padded
    corner = np.array([T.CORNERS[b] for b, _ in T.EDGES], np.int64)  # [12, 3]
    e_off = corner @ np.array([n1 * n2, n2, 1], np.int64)
    e_axis = np.array([a for _, a in T.EDGES], np.int64)
    valid = edges >= 0
    e = np.where(valid, edges, 0)
    slot = (base[:, None] + e_off[e]) * 3 + e_axis[e]
    faces = ids[slot][valid].reshape(-1, 3)
    return verts.reshape(-1, 3), faces.astype(np.int64)


def boundary_report(faces: np.ndarray):
    """(#directed edges that occur more than once, #directed edges whose reverse is missing)."""
    f = np.asarray(faces, np.int64)
    if len(f) == 0:
        return 0, 0
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key = d[:, 0] * (d.max() + 1) + d[:, 1]
    rkey = d[:, 1] * (d.max() + 1) + d[:, 0]
    uniq, cnt = np.unique(key, return_counts=True)
    return int((cnt > 1).sum()), int((~np.isin(rkey, uniq)).sum())


def euler_characteristic(verts: np.ndarray, faces: np.ndarray) -> int:
    f = np.asarray(faces, np.int64)
    d = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    n_edges = len(np.unique(d[:, 0] * len(verts) + d[:, 1]))
    return len(verts) - n_edges + len(f)
