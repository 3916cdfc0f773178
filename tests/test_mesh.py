"""CPU: the marching-cubes case table (neddf_b200/mc_table.py -> csrc/mc_table.cuh) and its numpy twin
(tests/mc_reference.py), which the GPU kernels are held to bit for bit in tests/test_mesh_gpu.py.

Mesh properties checked on the twin: closed, edge-manifold and consistently oriented surfaces on random volumes that
hit every case; the Euler characteristic, normal direction and interpolation error on analytic sphere and torus
volumes; non-finite corners, empty and minimal volumes; the PLY writer."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from neddf_b200 import mc_table as T
from tests import mc_reference as M

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def random_volumes():
    """Three 14^3 volumes of uniform values in [0, 1) bordered by one layer of outside values (threshold 0.5)."""
    out = []
    for seed in range(3):
        rng = np.random.default_rng(seed)
        v = np.ones((14, 14, 14), np.float32)
        v[1:-1, 1:-1, 1:-1] = rng.random((12, 12, 12), dtype=np.float32)
        out.append(v)
    return out


def sphere(shape=(16, 16, 16), center=(7.6, 7.3, 7.1), radius=5.3):
    g = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing="ij"), -1)
    d = g - np.array(center)
    return (np.linalg.norm(d, axis=-1) - radius).astype(np.float32), (center, radius)


def sphere_sdf(p, center, radius):
    d = p - np.array(center)
    n = np.linalg.norm(d, axis=-1)
    return n - radius, d / n[:, None]


def torus(shape=(22, 20, 12), center=(10.4, 9.7, 5.6), major=6.2, minor=2.6):
    g = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing="ij"), -1)
    return torus_sdf(g.reshape(-1, 3), center, major, minor)[0].reshape(shape).astype(np.float32), (center, major, minor)


def torus_sdf(p, center, major, minor):
    d = p - np.array(center)
    rho = np.hypot(d[:, 0], d[:, 1])
    q = np.stack([rho - major, d[:, 2]], 1)
    qn = np.linalg.norm(q, axis=1)
    grad = np.stack([q[:, 0] * d[:, 0] / rho, q[:, 0] * d[:, 1] / rho, q[:, 1]], 1) / qn[:, None]
    return qn - minor, grad


def analytic_volumes():
    """(name, volume, threshold) of every CPU volume the GPU test replays on the kernels."""
    vols = [(f"random{i}", v, 0.5) for i, v in enumerate(random_volumes())]
    vols.append(("sphere", sphere()[0], 0.0))
    vols.append(("sphere_noncubic", sphere((12, 17, 15), (5.7, 8.2, 7.4), 4.6)[0], 0.0))
    vols.append(("torus", torus()[0], 0.0))
    s = sphere()[0].copy()
    s[7, 7, 2] = np.nan
    s[3, 9, 8] = np.inf
    s[12, 6, 7] = -np.inf
    vols.append(("sphere_nonfinite", s, 0.0))
    vols.append(("all_inside", np.full((5, 6, 7), -1.0, np.float32), 0.0))
    vols.append(("all_outside", np.full((7, 5, 6), 1.0, np.float32), 0.0))
    vols.append(("cube2", np.array([[[-1, 1], [1, -1]], [[0.25, 2], [-3, 0.5]]], np.float32), 0.1))
    vols.append(("slab", np.random.default_rng(7).standard_normal((2, 9, 30)).astype(np.float32), 0.0))
    return vols


def face_normals(v, f):
    a, b, c = v[f[:, 0]].astype(np.float64), v[f[:, 1]].astype(np.float64), v[f[:, 2]].astype(np.float64)
    return np.cross(b - a, c - a), (a + b + c) / 3.0


def test_header_is_generator_output():
    r = subprocess.run([sys.executable, "-m", "neddf_b200.mc_table"], cwd=REPO, stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True, check=True)
    with open(os.path.join(REPO, "neddf_b200", "csrc", "mc_table.cuh")) as fh:
        assert fh.read() == r.stdout
    assert "820 triangles, at most 5 per case" in r.stderr


def test_table_properties():
    assert T.MAX_TRIS == 5 and T.TOTAL_TRIS == 820
    assert len(T.TABLE[0]) == 0 and len(T.TABLE[255]) == 0
    for case, tris in enumerate(T.TABLE):
        crossed = {e for e in range(12) if ((case >> T._edge_corners(e)[0]) & 1) != ((case >> T._edge_corners(e)[1]) & 1)}
        assert {e for t in tris for e in t} == crossed, case
        assert all(len(set(t)) == 3 for t in tris), case
        # every triangle side is a face segment (two crossings on one face) or a diagonal that lies in no face, and
        # within a case each directed side occurs once
        sides = [(t[q], t[(q + 1) % 3]) for t in tris for q in range(3)]
        assert len(sides) == len(set(sides)), case


def test_random_volumes_hit_every_case_and_close():
    seen = set()
    for v in random_volumes():
        seen |= set(np.unique(M.classify(v, 0.5)).tolist())
        verts, faces = M.marching_cubes(v, 0.5)
        assert len(faces) > 1000
        assert M.boundary_report(faces) == (0, 0)  # each directed edge once, its reverse once
        assert np.array_equal(np.unique(faces), np.arange(len(verts)))  # every vertex referenced
        assert np.isfinite(verts).all()
    assert seen == set(range(256))


@pytest.mark.parametrize("which", ["sphere", "sphere_noncubic", "torus"])
def test_analytic_surfaces(which):
    if which == "torus":
        vol, (center, major, minor) = torus()
        sdf = lambda p: torus_sdf(p, center, major, minor)  # noqa: E731
        chi, curv_r = 0, minor
    else:
        vol, (center, radius) = sphere() if which == "sphere" else sphere((12, 17, 15), (5.7, 8.2, 7.4), 4.6)
        sdf = lambda p: sphere_sdf(p, center, radius)  # noqa: E731
        chi, curv_r = 2, radius
    verts, faces = M.marching_cubes(vol, 0.0)
    assert M.boundary_report(faces) == (0, 0)
    assert M.euler_characteristic(verts, faces) == chi
    n, cen = face_normals(verts, faces)
    _, grad = sdf(cen)
    assert ((n * grad).sum(1) > 0).all()  # normals toward increasing value: outward for an SDF
    val, _ = sdf(verts.astype(np.float64))
    # linear interpolation along a grid edge (h = 1 in index space): |error| <= h^2 / 8 * max|f''| <= h^2 / (4 r)
    assert np.abs(val).max() <= 1.0 / (4 * curv_r) + 1e-5, float(np.abs(val).max())


def test_nonfinite_corners_emit_nothing():
    vol, _ = sphere()
    base_v, base_f = M.marching_cubes(vol, 0.0)
    s = dict((name, (v, t)) for name, v, t in analytic_volumes())["sphere_nonfinite"][0]
    verts, faces = M.marching_cubes(s, 0.0)
    case = M.classify(s, 0.0)
    bad = ~np.isfinite(s)
    touching = np.zeros(case.shape, bool)
    for di, dj, dk in T.CORNERS:
        touching |= bad[di:di + case.shape[0], dj:dj + case.shape[1], dk:dk + case.shape[2]]
    lost = M.TRI_COUNT[M.classify(vol, 0.0)[touching]].sum()
    assert lost > 0 and len(faces) == len(base_f) - lost
    assert np.isfinite(verts).all()
    assert np.array_equal(np.unique(faces), np.arange(len(verts)))  # no orphan vertex


@pytest.mark.parametrize("fill", [-1.0, 1.0])
def test_uniform_volume_is_empty(fill):
    verts, faces = M.marching_cubes(np.full((5, 6, 7), fill, np.float32), 0.0)
    assert verts.shape == (0, 3) and verts.dtype == np.float32
    assert faces.shape == (0, 3) and faces.dtype == np.int64


def test_single_cube_every_case():
    for case in range(256):
        v = np.ones((2, 2, 2), np.float32)
        for b, (i, j, k) in enumerate(T.CORNERS):
            if (case >> b) & 1:
                v[i, j, k] = -1.0
        verts, faces = M.marching_cubes(v, 0.0)
        assert len(faces) == len(T.TABLE[case])
        assert len(verts) == bin(T.EDGE_MASK[case]).count("1")
        if len(verts):
            assert set(np.unique(verts).tolist()) <= {0.0, 0.5, 1.0}  # t = 1/2 exactly


def test_vertex_arithmetic_is_float32():
    v = np.array([[[0.1, 0.7], [0.3, 0.9]], [[0.6, 0.2], [0.8, 0.05]]], np.float32)
    thr = 0.45
    verts, _ = M.marching_cubes(v, thr)
    lo, hi = v[0, 0, 0], v[1, 0, 0]
    t = (np.float32(thr) - lo) / (hi - lo)
    assert t.dtype == np.float32
    assert verts[0].tolist() == [np.float32(0.0) + t, 0.0, 0.0]


def test_write_ply_round_trip(tmp_path):
    from neddf_b200.mesh import read_ply, write_ply
    verts, faces = M.marching_cubes(torus()[0], 0.0)
    p = str(tmp_path / "t.ply")
    write_ply(p, verts, faces)
    with open(p, "rb") as fh:
        head = fh.read(200)
    assert head.startswith(b"ply\nformat binary_little_endian 1.0\nelement vertex ")
    assert b"property list uchar int vertex_indices\nend_header\n" in head
    v2, f2 = read_ply(p)
    assert np.array_equal(v2, verts) and np.array_equal(f2, faces)
    assert os.path.getsize(p) == len(head.split(b"end_header\n")[0]) + 11 + 12 * len(verts) + 13 * len(faces)
    write_ply(p, np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64))
    v3, f3 = read_ply(p)
    assert v3.shape == (0, 3) and f3.shape == (0, 3)


def test_marching_cubes_validates_inputs():
    from neddf_b200.mesh import marching_cubes
    with pytest.raises(ValueError, match="CUDA"):
        marching_cubes(torch.zeros(4, 4, 4), 0.0)
    with pytest.raises(TypeError):
        marching_cubes(np.zeros((4, 4, 4), np.float32), 0.0)
