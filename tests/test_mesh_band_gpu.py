"""GPU: narrow-band marching cubes (csrc/mcubes_band.cu behind neddf_b200.mesh.narrow_band_marching_cubes and
extract_mesh(..., lipschitz=L)).

- The kernels equal the numpy twin (tests/mc_band_reference.py) bit for bit, in order, on every CPU test volume.
- extract_mesh with a band equals the dense extract_mesh (vertices, faces, normals, colours; torch.equal) on the bunny
  NeDDF distance and a NeuS golden sdf, once the premise is shown to hold on the dense volume for the L used.
- Analytic spheres and tori at 1024^3 and 2048^3, where no dense call exists: closed, edge-manifold meshes on the
  surface, with exactly the evaluations the two passes promise.
- The mesh command at 1024^3 with --lipschitz."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import mc_band_reference as B
from tests import mc_reference as M
from tests.test_mesh_band import VOLS
from tests.test_mesh_gpu import THR, bunny_render

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LADDER = (1.0, 1.5, 2.0, 3.0, 4.0)


class Counted:
    """evaluate(idx) of a device volume or an analytic field, counting the points it is asked for."""

    def __init__(self, fn):
        self.fn, self.points = fn, 0

    def __call__(self, idx):
        assert idx.dtype == torch.int32 and idx.is_cuda and idx.dim() == 2 and idx.shape[1] == 3
        self.points += idx.shape[0]
        return self.fn(idx.long())


def band_mc(vol: np.ndarray, thr, band, normals):
    from neddf_b200.mesh import narrow_band_marching_cubes
    d = torch.from_numpy(np.ascontiguousarray(vol)).to(DEV)
    ev = Counted(lambda i: d[i[:, 0], i[:, 1], i[:, 2]])
    return narrow_band_marching_cubes(ev, vol.shape[0], thr, float(band), normals=normals), ev.points


@pytest.mark.parametrize("name,vol,thr,band", VOLS, ids=[v[0] for v in VOLS])
def test_kernels_match_twin(name, vol, thr, band):
    (v, f, nrm), points = band_mc(vol, thr, band, True)
    tv, tf, tn = B.marching_cubes(vol, thr, band, normals=True)
    assert v.dtype == torch.float32 and f.dtype == torch.int64 and nrm.dtype == torch.float32
    assert torch.equal(v.cpu(), torch.from_numpy(tv)), name
    assert torch.equal(f.cpu(), torch.from_numpy(tf)), name
    assert torch.equal(nrm.cpu(), torch.from_numpy(tn)), name
    assert points == B.evaluations(vol, thr, band)
    (v2, f2), _ = band_mc(vol, thr, band, False)
    assert torch.equal(v, v2) and torch.equal(f, f2)  # normals leave vertices and faces as they are
    (v3, f3, n3), _ = band_mc(vol, thr, band, True)
    assert torch.equal(v, v3) and torch.equal(f, f3) and torch.equal(nrm, n3)  # deterministic


def test_a_narrow_band_drops_bricks_and_their_faces():
    """The x3 sphere with the band of L = 1 (premise broken): the kernels still equal the twin, which loses faces."""
    from tests.test_mesh_band import BAND_L1, sphere
    vol = sphere(64, 3.0)
    (v, f, nrm), _ = band_mc(vol, 0.0, BAND_L1, True)
    tv, tf, tn = B.marching_cubes(vol, 0.0, BAND_L1, normals=True)
    assert torch.equal(v.cpu(), torch.from_numpy(tv)) and torch.equal(f.cpu(), torch.from_numpy(tf))
    assert torch.equal(nrm.cpu(), torch.from_numpy(tn))
    assert len(f) < len(M.marching_cubes(vol, 0.0)[1])


def premise_holds(vol: torch.Tensor, thr: float, band: float) -> bool:
    """On the device: every brick holding an emitting cell of the dense volume passes the admission rule."""
    n = vol.shape[0]
    m = n - 1
    inside, finite = vol < thr, torch.isfinite(vol)
    any_in = torch.zeros(m, m, m, dtype=torch.bool, device=vol.device)
    all_in = torch.ones_like(any_in)
    all_fin = torch.ones_like(any_in)
    for di, dj, dk in M.T.CORNERS:
        s = (slice(di, di + m), slice(dj, dj + m), slice(dk, dk + m))
        any_in |= inside[s]
        all_in &= inside[s]
        all_fin &= finite[s]
    emit = all_fin & any_in & ~all_in
    nb = B.n_bricks(n)
    pad = torch.zeros(nb * 8, nb * 8, nb * 8, dtype=torch.bool, device=vol.device)
    pad[:m, :m, :m] = emit
    hot = pad.view(nb, 8, nb, 8, nb, 8).any(5).any(3).any(1)
    c = torch.from_numpy(B.corner_index(n)).to(vol.device)
    active = torch.from_numpy(B.active_bricks(vol[c][:, c][:, :, c].cpu().numpy(), thr, band)).to(vol.device)
    return bool((active | ~hot).all())


def smallest_rung(vol, thr, n, what):
    for lip in LADDER:
        if premise_holds(vol, thr, float(B.band_for(lip, n))):
            print(f"{what}: premise holds at L = {lip}")
            return lip
    pytest.fail(f"{what}: the premise holds for no L in {LADDER}")


def assert_band_equals_dense(net, field, thr, n, what):
    vol = net._grid_volume(field, 1.1, n)
    lip = smallest_rung(vol, thr, n, what)
    del vol
    dense = net.extract_mesh(field, thr, cube_range=1.1, cube_resolution=n, with_color=True)
    band = net.extract_mesh(field, thr, cube_range=1.1, cube_resolution=n, with_color=True, lipschitz=lip)
    assert len(dense[1]) > 0
    for name, a, b in zip(("vertices", "faces", "normals", "colors"), dense, band):
        assert torch.equal(a, b), f"{what}: {name}"
    v, f = net.extract_mesh(field, thr, cube_range=1.1, cube_resolution=n, lipschitz=lip)
    assert torch.equal(v, dense[0]) and torch.equal(f, dense[1])


@pytest.mark.parametrize("engine", ["fp32", "tc"])
@pytest.mark.parametrize("n", [64, 256, 512])
def test_extract_mesh_band_equals_dense_bunny(n, engine):
    net = bunny_render(engine)[0].get_network()
    assert_band_equals_dense(net, "distance", THR, n, f"bunny {engine} {n}^3")


def test_extract_mesh_band_equals_dense_neus():
    from tests.test_neus_gpu import build
    from tests.test_neus_oracle import NeusCase
    net = build(NeusCase("relu"))[0].get_network()
    n = 128
    thr = float(net._grid_volume("sdf", 1.1, n).median())
    assert_band_equals_dense(net, "sdf", thr, n, f"NeuS relu sdf at {thr:g}")


def sphere_sdf(p, c=(0.03, -0.02, 0.01), radius=0.5):
    return np.linalg.norm(p - np.array(c), axis=-1) - radius


def torus_sdf(p, c=(0.02, 0.01, -0.03), major=0.6, minor=0.2):
    d = p - np.array(c)
    return np.hypot(np.hypot(d[..., 0], d[..., 1]) - major, d[..., 2]) - minor


def torch_field(which, n):
    """The analytic SDF in fp32 on the device at grid points (i, j, k) -> (x, y, z) = -r + (i, j, k) h."""
    h = np.float32(2.2 / (n - 1))

    def f(idx):
        p = idx.float() * float(h) - 1.1
        if which == "sphere":
            d = p - torch.tensor([0.03, -0.02, 0.01], device=DEV)
            return torch.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]) - 0.5
        d = p - torch.tensor([0.02, 0.01, -0.03], device=DEV)
        rho = torch.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) - 0.6
        return torch.sqrt(rho * rho + d[:, 2] * d[:, 2]) - 0.2
    return f


@pytest.mark.parametrize("n", [1024, 2048])
@pytest.mark.parametrize("which", ["sphere", "torus"])
def test_analytic_surfaces_beyond_the_dense_limit(which, n):
    from neddf_b200.mesh import narrow_band_marching_cubes
    h = 2.2 / (n - 1)
    band = float(B.band_for(1.0, n))
    ev = Counted(torch_field(which, n))
    v, f = narrow_band_marching_cubes(ev, n, 0.0, band)
    nb = B.n_bricks(n)
    n_active, rest = divmod(ev.points - (nb + 1) ** 3, 729)
    assert rest == 0 and n_active > 0
    # the bricks the analytic SDF admits, in float64 (a relative 1e-6 covers the fp32 evaluation's rounding)
    sdf = sphere_sdf if which == "sphere" else torus_sdf
    c = -1.1 + B.corner_index(n) * h
    corners = sdf(np.stack(np.meshgrid(c, c, c, indexing="ij"), -1))
    admitted = int(B.active_bricks(corners, 0.0, band * (1 + 1e-6)).sum())
    assert n_active <= admitted
    print(f"{which} {n}^3: {ev.points} evaluations ({ev.points / n ** 3:.2%} of n^3), {n_active} active bricks "
          f"({admitted} admitted in float64), {len(v)} vertices, {len(f)} faces")
    vn, fn = v.cpu().numpy(), f.cpu().numpy()
    assert M.boundary_report(fn) == (0, 0)  # closed and edge-manifold
    assert M.euler_characteristic(vn, fn) == (2 if which == "sphere" else 0)
    assert np.array_equal(np.unique(fn), np.arange(len(vn)))
    world = -1.1 + vn.astype(np.float64) * h
    assert np.abs(sdf(world)).max() <= 1e-2 * h


def test_mesh_command_band_at_1024(tmp_path):
    import yaml

    from neddf_b200.mesh import read_ply
    _, c = bunny_render()
    run = tmp_path / "bunny_run"
    (run / ".hydra").mkdir(parents=True)
    (run / "models").mkdir()
    with open(run / ".hydra" / "config.yaml", "w") as fh:
        yaml.safe_dump({"render": c.render_cfg, "network": c.net_cfg}, fh)
    torch.save(c.state_dict(), run / "models" / "model_02000.pth")
    env = dict(os.environ)
    env["PYTHONPATH"] = REPO + os.pathsep + env.get("PYTHONPATH", "")
    r = subprocess.run([sys.executable, "-m", "neddf_b200.mesh", str(run), "--resolution", "1024", "--lipschitz", "1.0",
                        "--color"], cwd=REPO, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=1200)
    assert r.returncode == 0, r.stdout
    got = read_ply(str(run / "mesh" / "mesh_1024_threshold0.0275.ply"), attributes=True)
    assert len(got["faces"]) > 1000
    assert set(got) == {"vertices", "faces", "normals", "colors"}
    assert got["faces"].min() >= 0 and got["faces"].max() < len(got["vertices"])
    assert np.isfinite(got["vertices"]).all() and np.abs(got["vertices"]).max() <= 1.1
    assert np.allclose(np.linalg.norm(got["normals"], axis=1), 1.0, atol=1e-5)
