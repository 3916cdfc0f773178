"""Numpy twin of the narrow-band marching-cubes kernels (csrc/mcubes_band.cu), float32 arithmetic, built on
tests/mc_reference.py (case table, vertex rule, output order) and tests/mc_normals_reference.py (vertex normals).

The grid's cells are cut into bricks of 8^3 cells: brick b covers points [8b, min(8b + 8, n - 1)] on each axis.  A
brick is active if one of its 8 corner values is non-finite or all 8 satisfy |v - thr| <= band in float32
(``neddf_mcb_bricks``).  Only the cells of active bricks are classified; each is classified by the dense rule, so the
mesh is the dense twin's mesh of a case array in which every cell of an inactive brick is empty.  Vertices are
ordered by global (grid point, axis), faces by (global cube, table order), and the normal of a vertex sums the faces
of kept cells only (``neddf_mcb_count`` / ``_emit`` / ``_normals``).

``premise`` is the condition under which that mesh is the dense one: every brick holding an emitting cell of the
dense grid is active.
"""
import math

import numpy as np

from tests import mc_normals_reference as N
from tests import mc_reference as M

BRICK = 8


def n_bricks(n: int) -> int:
    return (n - 1 + BRICK - 1) // BRICK


def corner_index(n: int) -> np.ndarray:
    """Grid index of each brick corner along an axis: min(8c, n - 1), c in [0, nb]."""
    return np.minimum(BRICK * np.arange(n_bricks(n) + 1), n - 1)


def band_for(lipschitz: float, n: int, cube_range: float = 1.1) -> np.float32:
    """extract_mesh's admission distance: L sqrt(3) 8 h in float64, h = 2r / (n - 1), rounded to float32."""
    return np.float32(lipschitz * math.sqrt(3.0) * BRICK * (2.0 * cube_range / (n - 1)))


def active_bricks(corners: np.ndarray, thr: float, band: float) -> np.ndarray:
    """Active flag of every brick [nb, nb, nb] from the brick-corner values [(nb + 1)^3]."""
    c = np.asarray(corners, np.float32)
    m = c.shape[0] - 1
    nonfinite = np.zeros((m, m, m), bool)
    near = np.ones((m, m, m), bool)
    with np.errstate(invalid="ignore"):
        close = np.abs(c - np.float32(thr)) <= np.float32(band)
    for di, dj, dk in M.T.CORNERS:
        nonfinite |= ~np.isfinite(c[di:di + m, dj:dj + m, dk:dk + m])
        near &= close[di:di + m, dj:dj + m, dk:dk + m]
    return nonfinite | near


def brick_of_cells(n: int) -> np.ndarray:
    """Brick index along an axis of every cell [n - 1]."""
    return np.arange(n - 1) // BRICK


def cell_mask(active: np.ndarray, n: int) -> np.ndarray:
    """Cells [n-1]^3 that lie in an active brick."""
    b = brick_of_cells(n)
    return active[np.ix_(b, b, b)]


def bricks(vol: np.ndarray, thr: float, band: float) -> np.ndarray:
    """Active flags [nb]^3 of a dense cubic volume, from its brick-corner values (the coarse pass)."""
    v = np.asarray(vol, np.float32)
    c = corner_index(v.shape[0])
    return active_bricks(v[np.ix_(c, c, c)], thr, band)


def evaluations(vol: np.ndarray, thr: float, band: float) -> int:
    """Points the two passes evaluate: (nb + 1)^3 corners plus 729 per active brick."""
    n = np.asarray(vol).shape[0]
    return (n_bricks(n) + 1) ** 3 + 729 * int(bricks(vol, thr, band).sum())


def premise(vol: np.ndarray, thr: float, band: float) -> bool:
    """Every brick that holds an emitting cell of the dense grid passes the admission rule."""
    v = np.asarray(vol, np.float32)
    n = v.shape[0]
    emit = M.TRI_COUNT[M.classify(v, thr)] > 0
    nb = n_bricks(n)
    hot = np.zeros((nb, nb, nb), bool)
    b = brick_of_cells(n)
    ii, jj, kk = np.nonzero(emit)
    hot[b[ii], b[jj], b[kk]] = True
    return bool((bricks(v, thr, band) | ~hot).all())


def cases(vol: np.ndarray, thr: float, band: float) -> np.ndarray:
    """Case byte of every cube [n-1]^3: the dense one in active bricks, 0 elsewhere."""
    v = np.asarray(vol, np.float32)
    case = M.classify(v, thr)
    case[~cell_mask(bricks(v, thr, band), v.shape[0])] = 0
    return case


def mesh_from_cases(vol: np.ndarray, thr: float, case: np.ndarray):
    """mc_reference.marching_cubes with the case array given: (vertices, faces, edge slots of the vertices)."""
    v = np.ascontiguousarray(vol, np.float32)
    n0, n1, n2 = v.shape
    thr32 = np.float32(thr)
    emit = M.TRI_COUNT[case] > 0
    flags = np.zeros((n0, n1, n2, 3), bool)
    for e, (b, axis) in enumerate(M.T.EDGES):
        di, dj, dk = M.T.CORNERS[b]
        flags[di:di + n0 - 1, dj:dj + n1 - 1, dk:dk + n2 - 1, axis] |= emit & (((M.EDGE_MASK[case] >> e) & 1) == 1)
    flat = flags.reshape(-1)
    ids = np.cumsum(flat, dtype=np.int64) - flat
    slots = np.nonzero(flat)[0]
    g, axis = slots // 3, slots % 3
    vf = v.reshape(-1)
    v0, v1 = vf[g], vf[g + np.array([n1 * n2, n2, 1], np.int64)[axis]]
    with np.errstate(divide="ignore", invalid="ignore"):
        t = (thr32 - v0) / (v1 - v0)
    verts = np.stack(np.unravel_index(g, (n0, n1, n2)), 1).astype(np.float32)
    rows = np.arange(len(slots))
    verts[rows, axis] = verts[rows, axis] + t
    cubes = np.nonzero(emit.reshape(-1))[0]
    ci, cj, ck = np.unravel_index(cubes, case.shape)
    base = (ci * n1 + cj) * n2 + ck
    edges = M.TRI_EDGES[case.reshape(-1)[cubes]]
    corner = np.array([M.T.CORNERS[b] for b, _ in M.T.EDGES], np.int64)
    e_off = corner @ np.array([n1 * n2, n2, 1], np.int64)
    e_axis = np.array([a for _, a in M.T.EDGES], np.int64)
    valid = edges >= 0
    e = np.where(valid, edges, 0)
    slot = (base[:, None] + e_off[e]) * 3 + e_axis[e]
    faces = ids[slot][valid].reshape(-1, 3).astype(np.int64)
    return verts.reshape(-1, 3), faces, slots


def vertex_normals(vol: np.ndarray, verts: np.ndarray, faces: np.ndarray, slots: np.ndarray) -> np.ndarray:
    """mc_normals_reference.vertex_normals over the band's faces; the fallback from the band's own edge slots."""
    v = np.ascontiguousarray(vol, np.float32)
    _, n1, n2 = v.shape
    acc = np.zeros((len(verts), 3), np.float32)
    np.add.at(acc, faces.reshape(-1), np.repeat(N.face_normals(verts, faces), 3, axis=0))
    x, y, z = acc[:, 0], acc[:, 1], acc[:, 2]
    length = np.sqrt((x * x + y * y) + z * z)
    with np.errstate(divide="ignore", invalid="ignore"):
        out = acc / length[:, None]
    g, axis = slots // 3, slots % 3
    vf = v.reshape(-1)
    upper = vf[g + np.array([n1 * n2, n2, 1], np.int64)[axis]]
    fallback = np.zeros((len(slots), 3), np.float32)
    fallback[np.arange(len(slots)), axis] = np.where(upper > vf[g], np.float32(1), np.float32(-1))
    zero = length == 0
    out[zero] = fallback[zero]
    return out.astype(np.float32)


def marching_cubes(vol: np.ndarray, thr: float, band: float, normals: bool = False):
    """(vertices, faces[, normals]) as neddf_b200.mesh.narrow_band_marching_cubes returns them for
    ``evaluate(i, j, k) = vol[i, j, k]`` on a cubic volume."""
    v = np.ascontiguousarray(vol, np.float32)
    assert v.shape[0] == v.shape[1] == v.shape[2]
    verts, faces, slots = mesh_from_cases(v, thr, cases(v, thr, band))
    if not normals:
        return verts, faces
    return verts, faces, vertex_normals(v, verts, faces, slots)
