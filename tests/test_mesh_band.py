"""CPU: the narrow-band marching-cubes twin (tests/mc_band_reference.py) against the dense twin, and the host-side
checks of the narrow band (extract_mesh(..., lipschitz=L), narrow_band_marching_cubes, the mesh command).

Wherever the premise holds (every brick holding an emitting cell passes the admission rule), the band twin must give
the dense twin's vertices, faces and normals in the same order; the GPU kernels are held to the band twin bit for bit
in tests/test_mesh_band_gpu.py.  A negative control shows the band being applied when the premise fails."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import mc_band_reference as B
from tests import mc_normals_reference as N
from tests import mc_reference as M

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = (2, 9, 10, 33, 50, 64)
BAND_L1 = np.float32(math.sqrt(3.0) * B.BRICK)  # L = 1 in index units (h = 1)


def grid(n):
    return np.stack(np.meshgrid(*[np.arange(n, dtype=np.float64)] * 3, indexing="ij"), -1)


def sphere(n, scale=1.0, center=(0.47, 0.52, 0.5), radius=0.33):
    d = grid(n) - np.array(center) * (n - 1)
    return (scale * (np.linalg.norm(d, axis=-1) - max(0.6, radius * (n - 1)))).astype(np.float32)


def torus(n):
    d = grid(n) - np.array([0.51, 0.48, 0.5]) * (n - 1)
    major, minor = max(0.5, 0.3 * (n - 1)), max(0.3, 0.12 * (n - 1))
    return (np.hypot(np.hypot(d[..., 0], d[..., 1]) - major, d[..., 2]) - minor).astype(np.float32)


def two_spheres(n, gap):
    a = np.linalg.norm(grid(n) - np.array([0.3, 0.45, 0.5]) * (n - 1), axis=-1) - 0.22 * (n - 1)
    b = np.linalg.norm(grid(n) - np.array([0.7 + gap, 0.55, 0.48]) * (n - 1), axis=-1) - 0.2 * (n - 1)
    return np.minimum(a, b).astype(np.float32)


def band_volumes():
    """(name, volume, threshold, band) on which the premise holds: the CPU and GPU tests replay all of them."""
    out = []
    for n in SIZES:
        out.append((f"sphere{n}", sphere(n), 0.0, BAND_L1))
        out.append((f"torus{n}", torus(n), 0.0, BAND_L1))
        out.append((f"sphere_x3_{n}", sphere(n, 3.0), 0.0, np.float32(3 * BAND_L1)))
        out.append((f"spheres_apart{n}", two_spheres(n, 0.1), 0.0, BAND_L1))
        out.append((f"spheres_overlap{n}", two_spheres(n, -0.15), 0.0, BAND_L1))
    s = sphere(50).copy()
    s[8, 24, 24] = np.nan  # on a brick corner near the surface
    s[20, 9, 30] = np.inf
    s[41, 25, 19] = -np.inf
    s[25, 25, 25] = np.nan  # deep inside: its brick is inactive
    out.append(("sphere_nonfinite50", s, 0.0, BAND_L1))
    s = sphere(33).copy()
    s[:, :, 30:] = np.nan  # a non-finite slab: every brick touching it is active and its cells emit nothing
    out.append(("sphere_nanslab33", s, 0.0, BAND_L1))
    out.append(("inside33", np.full((33, 33, 33), -1.0, np.float32), 0.0, BAND_L1))
    out.append(("outside10", np.full((10, 10, 10), 1.0, np.float32), 0.0, np.float32(0.5)))
    # integer centre and radius: grid values exactly on the level (t = 0 or 1 merges vertices)
    d = grid(41) - 20.0
    out.append(("sphere_on_grid41", (np.linalg.norm(d, axis=-1) - 12.0).astype(np.float32), 0.0, BAND_L1))
    out.append(("plane_on_grid17", (grid(17)[..., 0] - 8.0).astype(np.float32), 0.0, BAND_L1))
    return out


VOLS = band_volumes()


@pytest.mark.parametrize("name,vol,thr,band", VOLS, ids=[v[0] for v in VOLS])
def test_band_twin_equals_dense_twin(name, vol, thr, band):
    assert B.premise(vol, thr, band), name
    v, f, nrm = B.marching_cubes(vol, thr, band, normals=True)
    dv, df = M.marching_cubes(vol, thr)
    dn = N.vertex_normals(vol, thr, dv, df)[0]
    assert v.dtype == np.float32 and f.dtype == np.int64 and nrm.dtype == np.float32
    assert np.array_equal(v, dv) and np.array_equal(f, df), name
    assert np.array_equal(nrm, dn, equal_nan=True), name
    n = vol.shape[0]
    evals = B.evaluations(vol, thr, band)
    assert (B.n_bricks(n) + 1) ** 3 <= evals <= (B.n_bricks(n) + 1) ** 3 + 729 * B.n_bricks(n) ** 3


def test_sizes_cover_partial_and_single_bricks():
    assert B.n_bricks(2) == 1 and B.n_bricks(9) == 1 and B.n_bricks(10) == 2
    assert [(n - 1) % B.BRICK for n in SIZES] == [1, 0, 1, 0, 1, 7]
    assert B.corner_index(10).tolist() == [0, 8, 9] and B.corner_index(9).tolist() == [0, 8]


def test_the_band_skips_empty_space():
    vol = sphere(64)
    active = B.bricks(vol, 0.0, BAND_L1)
    assert 0 < active.sum() < active.size
    assert len(M.marching_cubes(vol, 0.0)[1]) > 1000
    assert B.evaluations(vol, 0.0, BAND_L1) < 64 ** 3


def test_nonfinite_corners_make_a_brick_active():
    corners = np.ones((3, 3, 3), np.float32)
    assert not B.active_bricks(corners, 0.0, 0.5).any()
    corners[2, 2, 2] = np.nan
    assert B.active_bricks(corners, 0.0, 0.5).tolist() == [[[False, False], [False, False]],
                                                           [[False, False], [False, True]]]
    assert B.active_bricks(np.zeros((2, 2, 2), np.float32), 0.0, 0.0).all()  # |v - thr| <= band, inclusive


def test_broken_premise_loses_faces():
    """The x3 sphere is 3-Lipschitz: with the band of L = 1 bricks on the surface fail the rule and lose their faces."""
    vol = sphere(64, 3.0)
    assert not B.premise(vol, 0.0, BAND_L1)
    v, f = B.marching_cubes(vol, 0.0, BAND_L1)
    dv, df = M.marching_cubes(vol, 0.0)
    assert len(f) < len(df) and len(v) < len(dv)
    assert B.premise(vol, 0.0, np.float32(3 * BAND_L1))


def test_band_for_extract_mesh():
    h = 2.2 / 511
    assert B.band_for(1.0, 512) == np.float32(math.sqrt(3.0) * 8 * h)
    assert B.band_for(2.0, 512) == np.float32(2 * math.sqrt(3.0) * 8 * h)


@pytest.mark.parametrize("lipschitz", [0.0, -1.0, float("nan"), float("inf"), -float("inf")])
def test_extract_mesh_rejects_bad_lipschitz(lipschitz):
    import neddf_b200
    with pytest.raises(ValueError, match="lipschitz"):
        neddf_b200.NeDDF().extract_mesh("distance", 0.0275, cube_resolution=64, lipschitz=lipschitz)


def test_extract_mesh_resolution_limits():
    import neddf_b200
    net = neddf_b200.NeDDF()
    with pytest.raises(ValueError, match="2048"):
        net.extract_mesh("distance", 0.0275, cube_resolution=2049, lipschitz=1.0)
    with pytest.raises(ValueError, match="lipschitz"):
        net.extract_mesh("distance", 0.0275, cube_resolution=513)


@pytest.mark.parametrize("net_name,field", [("NeRF", "density"), ("NeDDF", "density"), ("NeDDF", "aux_grad"),
                                            ("NeuS", "density")])
def test_extract_mesh_band_needs_the_distance_field(net_name, field):
    import neddf_b200
    with pytest.raises(ValueError, match="distance field"):
        getattr(neddf_b200, net_name)().extract_mesh(field, 0.5, cube_resolution=64, lipschitz=1.0)


def test_narrow_band_marching_cubes_validates_inputs():
    from neddf_b200.mesh import narrow_band_marching_cubes

    def f(idx):
        raise AssertionError("not evaluated")

    for n in (1, 2049, 64.0, True):
        with pytest.raises(ValueError, match="n must be"):
            narrow_band_marching_cubes(f, n, 0.0, 1.0)
    for band in (-1.0, float("nan"), float("inf"), 1e39):
        with pytest.raises(ValueError, match="band"):
            narrow_band_marching_cubes(f, 64, 0.0, band)
    with pytest.raises(ValueError, match="threshold"):
        narrow_band_marching_cubes(f, 64, float("nan"), 1.0)
    with pytest.raises(TypeError):
        narrow_band_marching_cubes(None, 64, 0.0, 1.0)


def test_mesh_command_above_512_needs_lipschitz(tmp_path):
    r = subprocess.run([sys.executable, "-m", "neddf_b200.mesh", str(tmp_path), "--resolution", "1024"], cwd=REPO,
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode != 0
    assert "--lipschitz" in r.stderr and "512" in r.stderr
    h = subprocess.run([sys.executable, "-m", "neddf_b200.mesh", "--help"], cwd=REPO, stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True, check=True)
    assert "--lipschitz" in h.stdout and "2048" in h.stdout
