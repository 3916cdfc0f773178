"""GPU: the vertex-normal kernel (csrc/mcubes.cu, neddf_mc_normals behind marching_cubes(..., normals=True)) against
its numpy twin (tests/mc_normals_reference.py) bit for bit; extract_mesh(..., with_color=True) on NeDDF (all three
engines), NeRF and NeuS against the kernels and one direct forward call; the orientation of the bunny's normals
against the field's gradient; `python -m neddf_b200.mesh RUN_DIR --color`."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import mc_normals_reference as N
from tests.test_mesh_gpu import THR, bunny_render, networks
from tests.test_mesh_normals import normal_volumes

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gpu_mc(vol: np.ndarray, thr: float, normals: bool):
    from neddf_b200.mesh import marching_cubes
    return marching_cubes(torch.from_numpy(np.ascontiguousarray(vol)).to(DEV), thr, normals=normals)


def assert_normals_equal_twin(vol, thr, what):
    v, f, n = gpu_mc(vol, thr, True)
    tv, tf, tn = N.marching_cubes(vol, thr)
    assert n.dtype == torch.float32 and n.shape == v.shape and n.is_cuda
    assert torch.equal(v.cpu(), torch.from_numpy(tv)) and torch.equal(f.cpu(), torch.from_numpy(tf)), what
    assert torch.equal(n.cpu(), torch.from_numpy(tn)), (what, float((n.cpu() - torch.from_numpy(tn)).abs().max()))
    v0, f0 = gpu_mc(vol, thr, False)
    assert torch.equal(v, v0) and torch.equal(f, f0), what  # normals=True leaves the mesh as it is
    v2, f2, n2 = gpu_mc(vol, thr, True)
    assert torch.equal(v, v2) and torch.equal(f, f2) and torch.equal(n, n2), what  # deterministic
    return v, f, n


@pytest.mark.parametrize("name,vol,thr", normal_volumes(), ids=[n for n, _, _ in normal_volumes()])
def test_normals_match_twin(name, vol, thr):
    v, _, n = assert_normals_equal_twin(vol, thr, name)
    if name.startswith("all_"):
        assert n.shape == (0, 3)
    if name in ("quantised", "cube_at_threshold"):
        tv, tf = N.M.marching_cubes(vol, thr)
        assert N.vertex_normals(vol, thr, tv, tf)[1].any()  # the fallback fired, and the kernel agreed


def test_normals_large_volume():
    """The 200 x 160 x 96 noisy volume of test_mesh_gpu.py: many blocks, long face lists."""
    rng = np.random.default_rng(5)
    g = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float32) for n in (200, 160, 96)], indexing="ij"), -1)
    vol = (np.sin(g[..., 0] * 0.21) + np.cos(g[..., 1] * 0.17) * np.sin(g[..., 2] * 0.13)).astype(np.float32)
    vol += 0.05 * rng.standard_normal(vol.shape).astype(np.float32)
    _, f, _ = assert_normals_equal_twin(vol, 0.1, "large")
    assert len(f) > 100000


def test_normals_entry_validates():
    from neddf_b200 import _lib as L
    lib = L.lib()
    vol = torch.zeros(4, 4, 4, device=DEV)
    ws = torch.empty(L.check(lib.neddf_mc_workspace_bytes(4, 4, 4)) + 256, dtype=torch.uint8, device=DEV)
    s = L.stream_ptr(DEV)
    assert lib.neddf_mc_normals(L.ptr(vol), 1, 4, 4, 0.0, L.ptr(ws), None, None, None, s) == -1
    assert lib.neddf_mc_normals(L.ptr(vol), 4, 4, 513, 0.0, L.ptr(ws), None, None, None, s) == -3
    assert lib.neddf_mc_normals(L.ptr(vol), 4, 4, 4, float("nan"), L.ptr(ws), None, None, None, s) == -1
    assert lib.neddf_mc_normals(L.ptr(vol), 4, 4, 4, 0.0, None, None, None, None, s) == -1
    import ctypes as C
    assert lib.neddf_mc_normals(L.ptr(vol), 4, 4, 4, 0.0, C.c_void_p(ws.data_ptr() + 16), None, None, None, s) == -1
    assert b"aligned" in lib.neddf_last_error()


# ------------------------------------------------------------------------------------------------- extract_mesh --
def direct_colors(net, points, view_dir):
    """One forward call over all vertices: what the chunked colour pass must reproduce bit for bit."""
    from neddf_b200 import Sampling
    with torch.no_grad():
        p = points[None]
        return net.forward(Sampling(p, view_dir[None].contiguous(), torch.zeros_like(p)))["color"][0]


def test_extract_mesh_with_color():
    """The networks of test_mesh_gpu.py: the bunny and a seeded default NeDDF on each engine, NeRF, NeuS."""
    from neddf_b200.mesh import marching_cubes
    for name, net, field in networks():
        r, n = 1.1, 40
        vol = net._grid_volume(field, r, n)
        thr = THR if name.startswith("bunny") else float(vol.median())
        wv, wf = net.extract_mesh(field, thr, cube_range=r, cube_resolution=n)
        cv, cf, cn, cc = net.extract_mesh(field, thr, cube_range=r, cube_resolution=n, with_color=True)
        assert len(wf) > 0, name
        assert torch.equal(cv, wv) and torch.equal(cf, wf), name
        _, _, index_normals = marching_cubes(vol, thr, normals=True)
        assert torch.equal(cn, index_normals[:, [2, 0, 1]]), name
        assert cc.dtype == torch.float32 and cc.shape == cv.shape and cc.device == cv.device, name
        view = -cn if field in ("distance", "sdf") else cn  # NeRF density grows inward
        ref = direct_colors(net, cv, view)
        assert torch.equal(cc, ref), (name, float((cc - ref).abs().max()))
        assert bool(torch.isfinite(cc).all()), name
        # the colour pass in many small chunks: each sample is its own column of the field kernels
        assert torch.equal(net._vertex_colors(cv, view, chunk=97), ref), name


def test_with_color_rejects_unsupported_fields():
    _, nerf, _ = next(x for x in networks() if x[0] == "nerf-relu")
    _, neus, _ = next(x for x in networks() if x[0] == "neus-relu")
    bunny = bunny_render()[0].get_network()
    for net, field in ((neus, "density"), (bunny, "aux_grad"), (nerf, "color")):
        with pytest.raises(ValueError, match="with_color"):
            net.extract_mesh(field, 0.0, cube_resolution=16, with_color=True)


def test_bunny_normals_follow_field_gradient():
    """The mesh normals against the device field's central-difference gradient (step h/4) at every vertex."""
    from neddf_b200 import Sampling
    render, _ = bunny_render()
    net = render.get_network()
    r, n = 1.1, 128
    v, f, nrm, _ = net.extract_mesh("distance", THR, cube_range=r, cube_resolution=n, with_color=True)
    step = 2 * r / (n - 1) / 4
    one_dir = torch.tensor([1.0, 0.0, 0.0], device=DEV).expand(len(v), 3)[None].contiguous()

    def dist(p):
        with torch.no_grad():
            return net.forward(Sampling(p[None].contiguous(), one_dir, torch.zeros_like(p[None])))["distance"][0].double()

    grad = torch.stack([dist(v + step * e) - dist(v - step * e) for e in torch.eye(3, device=DEV)], 1)
    grad = grad / grad.norm(dim=1, keepdim=True)
    cos = (nrm.double() * grad).sum(1).clamp(-1, 1)
    agree = float((cos > 0).double().mean())
    angle = float(torch.rad2deg(torch.acos(cos)).median())
    print(f"bunny distance {THR} at {n}^3: {len(v)} vertices, sign agreement {agree:.4%}, median angle {angle:.2f} deg")
    assert agree >= 0.99, agree


def test_auto_engine_recolours_on_fp32_after_leaving_fp16_range():
    """A colour trunk blown past fp16 range (as test_gpu_parity.py's engine-cliff test does): engine "auto" warns,
    switches the network to fp32 and evaluates the colours again, so they are the fp32 engine's bit for bit; the
    geometry, which the colour trunk does not touch, is what extract_mesh gives."""
    render, _ = bunny_render("auto")
    net = render.get_network()
    with torch.no_grad():
        net.layers_col[0].weight.mul_(1e5)
    assert net.resolved_engine() == "tc"
    v0, f0 = net.extract_mesh("distance", THR, cube_resolution=40)
    with pytest.warns(RuntimeWarning, match="fp16 range"):
        v, f, nrm, col = net.extract_mesh("distance", THR, cube_resolution=40, with_color=True)
    assert net.resolved_engine() == "fp32"
    assert torch.equal(v, v0) and torch.equal(f, f0)
    render.set_engine("fp32")
    ref = direct_colors(net, v, -nrm)
    assert torch.equal(col, ref) and bool(torch.isfinite(col).all())
    assert float(col.abs().max()) > 1e3  # out of fp16 territory indeed


def test_mesh_command_writes_colors(tmp_path):
    import yaml

    from neddf_b200.eval_io import color_to_uint8
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
    r = subprocess.run([sys.executable, "-m", "neddf_b200.mesh", str(run), "--resolution", "40", "--color"], cwd=REPO,
                       env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout
    got = read_ply(str(run / "mesh" / "mesh_40_threshold0.0275.ply"), attributes=True)
    wv, wf, wn, wc = render.get_network().extract_mesh("distance", THR, cube_range=1.1, cube_resolution=40,
                                                       with_color=True)
    assert len(wf) > 0
    assert np.array_equal(got["vertices"], wv.cpu().numpy()) and np.array_equal(got["faces"], wf.cpu().numpy())
    assert np.array_equal(got["normals"], wn.cpu().numpy())
    assert np.array_equal(got["colors"], color_to_uint8(wc).cpu().numpy())
    assert len(np.unique(got["colors"].reshape(-1, 3), axis=0)) > 1
