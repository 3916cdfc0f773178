"""Numpy twin of the vertex-normal kernel (csrc/mcubes.cu, mc_normals), built on the output of tests/mc_reference.py.

A vertex normal is the sum of the unnormalised face normals (v1 - v0) x (v2 - v0) of the faces that use the vertex,
in ascending face index, normalised.  Every float32 step is rounded on its own, as the kernel's ``__fsub_rn`` /
``__fmul_rn`` / ``__fadd_rn`` / ``__fsqrt_rn`` / ``__fdiv_rn`` are: numpy float32 ufuncs round each operation and
never contract a multiply and an add.  ``np.add.at`` over the face corners interleaved in face order
([f0c0, f0c1, f0c2, f1c0, ...]) adds each vertex's terms in ascending face index, starting from +0.  A zero-length sum
falls back to the vertex's edge axis, signed toward the edge corner with the larger value.
"""
import numpy as np

from tests import mc_reference as M


def edge_slots(vol: np.ndarray, thr: float) -> np.ndarray:
    """Edge slot (grid point linear index * 3 + axis) of every vertex, in vertex id order."""
    v = np.asarray(vol, np.float32)
    n0, n1, n2 = v.shape
    case = M.classify(v, thr)
    emit = M.TRI_COUNT[case] > 0
    flags = np.zeros((n0, n1, n2, 3), bool)
    for e, (b, axis) in enumerate(M.T.EDGES):
        di, dj, dk = M.T.CORNERS[b]
        flags[di:di + n0 - 1, dj:dj + n1 - 1, dk:dk + n2 - 1, axis] |= emit & (((M.EDGE_MASK[case] >> e) & 1) == 1)
    return np.nonzero(flags.reshape(-1))[0]


def face_normals(verts: np.ndarray, faces: np.ndarray) -> np.ndarray:
    """Unnormalised float32 face normals [F,3], each subtraction and product rounded on its own."""
    v = np.asarray(verts, np.float32)
    f = np.asarray(faces, np.int64)
    p0, p1, p2 = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    a, b = p1 - p0, p2 - p0
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1],
                     a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                     a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1).astype(np.float32)


def fallback_normals(vol: np.ndarray, thr: float) -> np.ndarray:
    """The fallback of every vertex [V,3]: its edge axis, signed toward the edge corner with the larger value."""
    v = np.ascontiguousarray(vol, np.float32)
    n0, n1, n2 = v.shape
    slots = edge_slots(v, thr)
    g, axis = slots // 3, slots % 3
    vf = v.reshape(-1)
    upper = vf[g + np.array([n1 * n2, n2, 1], np.int64)[axis]]
    out = np.zeros((len(slots), 3), np.float32)
    out[np.arange(len(slots)), axis] = np.where(upper > vf[g], np.float32(1), np.float32(-1))
    return out


def vertex_normals(vol: np.ndarray, thr: float, verts: np.ndarray, faces: np.ndarray):
    """(normals [V,3] float32, fallback [V] bool) for the mesh that ``mc_reference.marching_cubes(vol, thr)``
    returned, as neddf_b200.mesh.marching_cubes(..., normals=True) computes them."""
    f = np.asarray(faces, np.int64)
    acc = np.zeros((len(verts), 3), np.float32)
    np.add.at(acc, f.reshape(-1), np.repeat(face_normals(verts, f), 3, axis=0))
    x, y, z = acc[:, 0], acc[:, 1], acc[:, 2]
    length = np.sqrt((x * x + y * y) + z * z)
    fallback = length == 0
    with np.errstate(divide="ignore", invalid="ignore"):
        out = acc / length[:, None]
    out[fallback] = fallback_normals(vol, thr)[fallback]
    return out.astype(np.float32), fallback


def marching_cubes(vol: np.ndarray, thr: float):
    """(vertices, faces, normals) as neddf_b200.mesh.marching_cubes(volume, thr, normals=True) returns them."""
    verts, faces = M.marching_cubes(vol, thr)
    return verts, faces, vertex_normals(vol, thr, verts, faces)[0]
