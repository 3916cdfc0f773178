"""GPU: the marching-cubes kernels (csrc/mcubes.cu behind neddf_b200.mesh.marching_cubes) against their numpy twin
(tests/mc_reference.py) bit for bit, the device grid behind voxelize / extract_mesh against the host grid it
replaces and against the reference's own voxelize (golden case_mesh_bunny.npz), the world mapping of extract_mesh,
and the `python -m neddf_b200.mesh` command."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import mc_reference as M
from tests.helpers import GOLDEN, PARITY_TOL, Case, nerr
from tests.test_mesh import analytic_volumes

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
THR = 0.0275  # the reference visualiser's iso-level of the NeDDF distance field


def gpu_mc(vol: np.ndarray, thr: float):
    from neddf_b200.mesh import marching_cubes
    return marching_cubes(torch.from_numpy(np.ascontiguousarray(vol)).to(DEV), thr)


def assert_equal_to_twin(vol, thr, what):
    v, f = gpu_mc(vol, thr)
    tv, tf = M.marching_cubes(vol, thr)
    assert v.dtype == torch.float32 and f.dtype == torch.int64 and v.shape[1] == 3 and f.shape[1] == 3
    assert torch.equal(v.cpu(), torch.from_numpy(tv)), what
    assert torch.equal(f.cpu(), torch.from_numpy(tf)), what
    return v, f


@pytest.mark.parametrize("name,vol,thr", analytic_volumes(), ids=[n for n, _, _ in analytic_volumes()])
def test_marching_cubes_matches_twin(name, vol, thr):
    v, f = assert_equal_to_twin(vol, thr, name)
    v2, f2 = gpu_mc(vol, thr)
    assert torch.equal(v, v2) and torch.equal(f, f2)  # deterministic
    if name.startswith("all_"):
        assert v.shape == (0, 3) and f.shape == (0, 3)


def test_marching_cubes_large_volume_deterministic():
    """A 200 x 160 x 96 noisy volume: many blocks per launch, multi-tile scans."""
    rng = np.random.default_rng(5)
    g = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float32) for n in (200, 160, 96)], indexing="ij"), -1)
    vol = (np.sin(g[..., 0] * 0.21) + np.cos(g[..., 1] * 0.17) * np.sin(g[..., 2] * 0.13)).astype(np.float32)
    vol += 0.05 * rng.standard_normal(vol.shape).astype(np.float32)
    v, f = assert_equal_to_twin(vol, 0.1, "large")
    assert len(f) > 100000
    v2, f2 = gpu_mc(vol, 0.1)
    assert torch.equal(v, v2) and torch.equal(f, f2)


def test_marching_cubes_rejects_bad_input():
    from neddf_b200.mesh import marching_cubes
    bad = [(torch.zeros(4, 4, 4, device=DEV, dtype=torch.float64), 0.0), (torch.zeros(4, 4, device=DEV), 0.0),
           (torch.zeros(4, 4, 4, device=DEV).transpose(0, 2), 0.0), (torch.zeros(1, 4, 4, device=DEV), 0.0),
           (torch.zeros(2, 2, 513, device=DEV), 0.0), (torch.zeros(4, 4, 4, device=DEV), float("nan")),
           (torch.zeros(4, 4, 4, device=DEV), 1e39)]
    for vol, thr in bad:
        with pytest.raises(ValueError):
            marching_cubes(vol, thr)
    from neddf_b200 import _lib as L
    lib = L.lib()
    assert lib.neddf_mc_workspace_bytes(1, 4, 4) == -1
    assert lib.neddf_mc_workspace_bytes(4, 513, 4) == -3
    assert lib.neddf_mc_workspace_bytes(512, 512, 512) > 3 * 512 ** 3 * 4


# ---------------------------------------------------------------------------------------------------- device grid --
def host_voxelize(net, field_name, cube_range, cube_resolution, chunk=65536):
    """The host-meshgrid voxelize this project had before the device grid (base_neuralfield.py:49-79)."""
    from neddf_b200 import Sampling
    with torch.no_grad():
        ids = np.linspace(-cube_range, cube_range, cube_resolution)
        zs, ys, xs = np.meshgrid(ids, ids, ids)
        pos = torch.from_numpy(np.stack([xs.reshape(-1), ys.reshape(-1), zs.reshape(-1)], 1).astype(np.float32))
        n = cube_resolution ** 3
        result = np.zeros(n, np.float32)
        one_dir = torch.tensor([[1.0, 0.0, 0.0]])
        for i in range(0, n, chunk):
            j = min(n, i + chunk)
            p = pos[None, i:j, :].to(DEV)
            s = Sampling(p, one_dir.expand(j - i, -1)[None].to(DEV).contiguous(), torch.zeros_like(p))
            result[i:j] = net.forward(s)[field_name].view(-1).detach().cpu().numpy()
        return result.reshape(cube_resolution, cube_resolution, cube_resolution)


def bunny_render(engine="auto"):
    """The bunny checkpoint in constructor state (no set_iter), as the reference visualiser meshes it."""
    import neddf_b200
    c = Case("bunny")
    r = neddf_b200.NeRFRender(network_config=c.net_cfg, **{k: v for k, v in c.render_cfg.items() if k != "_target_"})
    r.load_state_dict(c.state_dict())
    r.to(DEV)
    r.set_engine(engine)
    return r, c


def networks():
    import tests.gpu_util as G
    from tests.test_nerf_gpu import build as build_nerf
    from tests.test_nerf_oracle import NerfCase
    from tests.test_neus_gpu import build as build_neus
    from tests.test_neus_oracle import NeusCase
    for engine in ("fp32", "tc", "tc2"):
        yield f"bunny-{engine}", bunny_render(engine)[0].get_network(), "distance"
        yield f"default-{engine}", G.build_render(Case("default"), engine).get_network(), "distance"
    yield "nerf-relu", build_nerf(NerfCase("relu"))[0].get_network(), "density"
    yield "neus-relu", build_neus(NeusCase("relu"))[0].get_network(), "sdf"


def test_device_grid_equals_host_grid():
    """Same points, same order, same values: every field kernel computes each sample as its own GEMM column, so
    neither the grid's construction nor the chunking may change a bit."""
    from neddf_b200.mesh import marching_cubes
    for name, net, field in networks():
        ref = host_voxelize(net, field, 1.1, 21)
        got = net.voxelize(field, cube_range=1.1, cube_resolution=21, chunk=1000)
        assert got.dtype == np.float32 and got.shape == (21, 21, 21)
        assert np.array_equal(got, ref), (name, float(np.abs(got - ref).max()))
        vol = net._grid_volume(field, 1.1, 21)
        assert vol.is_cuda and torch.equal(vol.cpu(), torch.from_numpy(ref)), name
        thr = float(np.median(ref))
        wv, wf = net.extract_mesh(field, thr, cube_range=1.1, cube_resolution=21)
        iv, f = marching_cubes(vol, thr)
        assert len(f) > 0 and torch.equal(wf, f), name
        tv, tf = M.marching_cubes(ref, thr)
        assert torch.equal(iv.cpu(), torch.from_numpy(tv)) and torch.equal(f.cpu(), torch.from_numpy(tf)), name


def golden_volume():
    z = np.load(os.path.join(GOLDEN, "case_mesh_bunny.npz"))
    return z["volume"], float(z["cube_range"]), int(z["cube_resolution"])


def test_bunny_grid_matches_reference_voxelize():
    gold, r, n = golden_volume()
    render, _ = bunny_render()
    net = render.get_network()
    got = net.voxelize("distance", cube_range=r, cube_resolution=n)
    assert nerr(got, gold) <= PARITY_TOL, nerr(got, gold)
    # the mesh of the device volume against the twin on the reference's volume: same case on every cube whose corners
    # all lie clear of the threshold, and on those cubes' edges a vertex shift within |dv| / |v_upper - v_lower|
    vol = net._grid_volume("distance", r, n)
    gv, gf = assert_equal_to_twin(vol.cpu().numpy(), THR, "bunny device volume")
    tv, tf = M.marching_cubes(gold, THR)
    assert len(gf) > 0 and len(tf) > 0
    mine = vol.cpu().numpy()
    margin = 1e-4 * float(np.abs(gold).max())
    clear = np.abs(gold - THR) > margin
    case_g, case_m = M.classify(gold, THR), M.classify(mine, THR)
    safe = np.ones(case_g.shape, bool)
    for di, dj, dk in M.T.CORNERS:
        safe &= clear[di:di + n - 1, dj:dj + n - 1, dk:dk + n - 1]
    assert safe.sum() > 0.99 * safe.size
    assert np.array_equal(case_g[safe], case_m[safe])
    ids_g, ids_m = slot_ids(gold, THR), slot_ids(mine, THR)
    checked = 0
    for c in zip(*np.nonzero(safe & (M.TRI_COUNT[case_g] > 0))):
        for e in range(12):
            if not (M.EDGE_MASK[case_g[c]] >> e) & 1:
                continue
            b, axis = M.T.EDGES[e]
            lo = tuple(int(x) + o for x, o in zip(c, M.T.CORNERS[b]))
            hi = tuple(x + (1 if a == axis else 0) for a, x in enumerate(lo))
            slot = (lo[0] * n * n + lo[1] * n + lo[2]) * 3 + axis
            dv = max(abs(float(mine[lo]) - float(gold[lo])), abs(float(mine[hi]) - float(gold[hi])))
            # exact for real-valued t; each of the two vertices adds its fp32 rounding (of t and of lower + t)
            bound = dv / abs(float(mine[hi]) - float(mine[lo])) + 2 * float(np.spacing(np.float32(n)))
            shift = np.abs(gv[ids_m[slot]].cpu().numpy().astype(np.float64) - tv[ids_g[slot]]).max()
            assert shift <= bound, (c, e, shift, bound)
            checked += 1
    assert checked > 0


def slot_ids(vol, thr):
    """Vertex id of every edge slot (valid where the slot is flagged), as the kernels number them."""
    n0, n1, n2 = vol.shape
    case = M.classify(vol, thr)
    emit = M.TRI_COUNT[case] > 0
    flags = np.zeros((n0, n1, n2, 3), bool)
    for e, (b, axis) in enumerate(M.T.EDGES):
        di, dj, dk = M.T.CORNERS[b]
        flags[di:di + n0 - 1, dj:dj + n1 - 1, dk:dk + n2 - 1, axis] |= emit & (((M.EDGE_MASK[case] >> e) & 1) == 1)
    flat = flags.reshape(-1)
    return np.cumsum(flat) - flat


def test_extract_mesh_world_mapping():
    from neddf_b200.mesh import marching_cubes
    render, _ = bunny_render()
    net = render.get_network()
    r, n = 1.1, 40
    wv, wf = net.extract_mesh("distance", THR, cube_range=r, cube_resolution=n)
    iv, f = marching_cubes(net._grid_volume("distance", r, n), THR)
    assert torch.equal(wf, f) and len(f) > 0
    h = 2 * r / (n - 1)
    iv64 = iv.cpu().double()
    ref = torch.stack([-r + iv64[:, 2] * h, -r + iv64[:, 0] * h, -r + iv64[:, 1] * h], 1)
    assert wv.dtype == torch.float32
    assert float((wv.cpu().double() - ref).abs().max()) <= 1e-6


def test_mesh_command_writes_ply(tmp_path):
    import yaml

    from neddf_b200.mesh import read_ply
    render, c = bunny_render()
    run = tmp_path / "bunny_run"
    (run / ".hydra").mkdir(parents=True)
    (run / "models").mkdir()
    with open(run / ".hydra" / "config.yaml", "w") as fh:
        yaml.safe_dump({"render": c.render_cfg, "network": c.net_cfg}, fh)
    torch.save(c.state_dict(), run / "models" / "model_02000.pth")
    env = dict(os.environ)
    env["PYTHONPATH"] = REPO + os.pathsep + env.get("PYTHONPATH", "")
    r = subprocess.run([sys.executable, "-m", "neddf_b200.mesh", str(run), "--resolution", "40"], cwd=REPO, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout
    path = run / "mesh" / "mesh_40_threshold0.0275.ply"
    assert path.exists(), r.stdout
    v, f = read_ply(str(path))
    wv, wf = render.get_network().extract_mesh("distance", THR, cube_range=1.1, cube_resolution=40)
    assert len(f) > 0
    assert np.array_equal(v, wv.cpu().numpy()) and np.array_equal(f, wf.cpu().numpy())
