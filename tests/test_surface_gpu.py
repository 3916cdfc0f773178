"""GPU: sphere tracing (csrc/surface.cu behind BaseNeuralField.trace_surface / NeRFRender.render_surface).

The kernels against the float32 twin (tests/trace_reference.py) bit for bit on analytic fields; the whole trace against
the twin driven by the same network; the bunny against the float64 oracle and against its extracted mesh; normals and
colours against direct forward calls; edge cases; the ``python -m neddf_b200.surface`` command."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import trace_reference as T
from tests.helpers import Case
from tests.test_surface import BUNNY_IMAGE, bunny_reference, fan

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATE_KEYS = ("t", "lo", "hi", "state", "steps")


def L():
    from neddf_b200 import _lib
    return _lib


# ------------------------------------------------------------------------------------- kernels against the twin --
def kernel_trace(field, d, o, near, far, level, max_steps):
    """init / step through the ABI with the field evaluated on the host from the kernels' packed samples."""
    lib, n = L().lib(), len(d)
    f32, i32 = dict(device=DEV, dtype=torch.float32), dict(device=DEV, dtype=torch.int32)
    rd, ro = torch.from_numpy(d).to(DEV), torch.from_numpy(o).to(DEV)
    t, lo, hi = (torch.empty(n, **f32) for _ in range(3))
    state, steps, count = torch.empty(n, **i32), torch.empty(n, **i32), torch.empty(1, **i32)
    live = [torch.empty(n, **i32), torch.empty(n, **i32)]
    pos, dirs = torch.empty(n, 3, **f32), torch.empty(n, 3, **f32)
    P = L().ptr
    s = L().stream_ptr(DEV)
    L().check(lib.neddf_trace_init(P(rd), P(ro), n, near, P(t), P(lo), P(hi), P(state), P(steps), P(live[0]), P(pos),
                                   P(dirs), s))
    counts, k, n_live = [], 0, n
    while n_live:
        v = torch.from_numpy(field(pos[:n_live].cpu().numpy(), dirs[:n_live].cpu().numpy())).to(DEV)
        L().check(lib.neddf_trace_step(P(v), P(live[k]), n_live, P(rd), P(ro), far, level, max_steps, P(t), P(lo), P(hi),
                                       P(state), P(steps), P(live[1 - k]), P(count), P(pos), P(dirs), s))
        k = 1 - k
        n_live = int(count.item())
        counts.append(n_live)
    out = dict(t=t, lo=lo, hi=hi, state=state, steps=steps)
    return {k_: v.cpu() for k_, v in out.items()}, counts, (rd, ro, t, state)


def kernel_normals(field, rd, ro, t, state):
    """trace_hits, fd_points, fd_normals through the ABI -> (hit ids, packed hit points, fd points, normals by ray)."""
    lib, n = L().lib(), rd.shape[0]
    P, s = L().ptr, L().stream_ptr(DEV)
    hits, count = torch.empty(n, device=DEV, dtype=torch.int32), torch.empty(1, device=DEV, dtype=torch.int32)
    pos, dirs = torch.empty(n, 3, device=DEV), torch.empty(n, 3, device=DEV)
    L().check(lib.neddf_trace_hits(P(rd), P(ro), n, P(t), P(state), P(hits), P(count), P(pos), P(dirs), s))
    m = int(count.item())
    pts, pd = torch.empty(6 * m, 3, device=DEV), torch.empty(6 * m, 3, device=DEV)
    L().check(lib.neddf_trace_fd_points(P(pos), P(dirs), m, P(pts), P(pd), s))
    v = torch.from_numpy(field(pts.cpu().numpy(), pd.cpu().numpy())).to(DEV)
    normal = torch.zeros(n, 3, device=DEV)
    L().check(lib.neddf_trace_fd_normals(P(v), P(pos), P(hits), m, P(normal), s))
    return hits[:m].cpu().long(), pos[:m].cpu(), pts.cpu(), normal.cpu()


def analytic_cases():
    a = math.radians(0.5)
    graze = (np.array([[math.cos(a), 0, -math.sin(a)]] * 3, np.float32), np.array([[0, 0, 1.0]] * 3, np.float32))
    yield "sphere", T.sphere_sdf((0, 0, 0), 1.0), fan(9, 0.5), 1.0, 8.0, 0.0, 128
    yield "sphere_level", T.sphere_sdf((0.1, -0.2, 0.3), 0.8), fan(9, 0.6), 1.0, 8.0, 0.05, 128
    yield "double_sdf", T.sphere_sdf((0, 0, 0), 1.0, scale=2.0), fan(9, 0.5), 2.5, 8.0, 0.0, 128
    yield "double_sdf_cut", T.sphere_sdf((0, 0, 0), 1.0, scale=2.0), fan(9, 0.5), 2.5, 8.0, 0.0, 6
    yield "misses", T.sphere_sdf((0, 0, 0), 1.0), fan(21, 3.0), 1.0, 8.0, 0.0, 128
    yield "inside", T.sphere_sdf((0, 0, -4), 1.0), fan(5, 0.2), 0.5, 8.0, 0.0, 128
    yield "grazing_plane", T.plane_sdf((0, 0, 1), 0.0), graze, 0.0, 1000.0, 0.0, 64


@pytest.mark.parametrize("case", list(analytic_cases()), ids=[c[0] for c in analytic_cases()])
def test_kernels_match_twin(case):
    name, field, (d, o), near, far, level, max_steps = case
    got, counts, dev = kernel_trace(field, d, o, near, far, level, max_steps)
    ref = T.trace(field, d, o, near, far, level, max_steps)
    for k in STATE_KEYS:
        assert torch.equal(got[k], torch.from_numpy(ref[k])), (name, k)
    assert counts == ref["live_counts"], name
    hits, pos, pts, normal = kernel_normals(field, *dev)
    want_hits = np.nonzero(ref["state"] == T.HIT)[0]
    assert sorted(hits.tolist()) == want_hits.tolist(), name
    tp = T.points(o[hits.numpy()], d[hits.numpy()], ref["t"][hits.numpy()])
    assert torch.equal(pos, torch.from_numpy(tp)), name
    tpts, tpd = T.fd_points(tp, d[hits.numpy()])
    assert torch.equal(pts, torch.from_numpy(tpts)), name
    tn = np.zeros((len(d), 3), np.float32)
    tn[hits.numpy()] = T.fd_normals(field(tpts, tpd), tp)
    assert torch.equal(normal, torch.from_numpy(tn)), name


# ---------------------------------------------------------------------------------------------- orchestration --
def bunny(engine="fp32"):
    import tests.gpu_util as G
    c = Case("bunny")
    return G.build_render(c, engine), G.build_camera(c)


def image_rays(render, cam, width, height, downsampling):
    from neddf_b200.render import _camera_host
    n = (width // downsampling) * (height // downsampling)
    rd, ro = torch.empty(n, 3, device=DEV), torch.empty(n, 3, device=DEV)
    L().check(L().lib().neddf_make_image_rays(width, height, downsampling, 0, n, *_camera_host(cam), L().ptr(rd),
                                              L().ptr(ro), L().stream_ptr(DEV)))
    return rd.cpu().numpy(), ro.cpu().numpy()


def net_field(net, key):
    from neddf_b200 import Sampling

    def f(p, d):
        pt = torch.from_numpy(p).to(DEV)[None]
        with torch.no_grad():
            return net.forward(Sampling(pt, torch.from_numpy(d).to(DEV)[None], torch.zeros_like(pt)))[key] \
                .reshape(-1).cpu().numpy()
    return f


def flat(img):
    return {k: v.reshape(-1, v.shape[-1]).squeeze(-1) if v.shape[-1] == 1 else v.reshape(-1, 3) for k, v in img.items()}


def check_against_twin(render, cam, key, level, image):
    net = render.get_network()
    img = render.render_surface(camera=cam, level=level, **image)
    w, h = image["width"] // image["downsampling"], image["height"] // image["downsampling"]
    assert img["depth"].shape == (h, w, 1) and img["hit"].dtype == torch.bool and img["steps"].dtype == torch.int32
    assert img["normal"].shape == (h, w, 3) and img["color"].shape == (h, w, 3)
    again = render.render_surface(camera=cam, level=level, **image)
    for k in img:
        assert torch.equal(img[k], again[k]), k
    d, o = image_rays(render, cam, **image)
    field = net_field(net, key)
    ref = T.trace(field, d, o, render.dist_near, render.dist_far, level, 128)
    got = {k: v.cpu() for k, v in flat(img).items()}
    assert torch.equal(got["depth"], torch.from_numpy(ref["t"]))
    assert torch.equal(got["steps"], torch.from_numpy(ref["steps"]))
    hit = ref["state"] == T.HIT
    assert torch.equal(got["hit"], torch.from_numpy(hit))
    print(f"\n[surface-twin] {key} level {level:.4f}: {int(hit.sum())} hits of {hit.size}")
    p = torch.from_numpy(T.points(o[hit], d[hit], ref["t"][hit])).to(DEV)
    dd = torch.from_numpy(d[hit]).to(DEV)
    return net, img, got, hit, p, dd, field


def test_render_surface_equals_twin_bunny():
    """fp32 engine: the twin fed by net.forward gives the same trace; colour and normal equal direct calls."""
    render, cam = bunny("fp32")
    net, img, got, hit, p, dd, field = check_against_twin(render, cam, "distance", 0.07, BUNNY_IMAGE)
    assert hit.sum() > 100
    from neddf_b200 import Sampling
    with torch.no_grad():
        col = net.forward(Sampling(p[None], dd[None], torch.zeros_like(p)[None]))["color"].reshape(-1, 3)
    assert torch.equal(got["color"][torch.from_numpy(hit)], col.cpu())
    assert torch.equal(got["color"][torch.from_numpy(~hit)], torch.zeros(int((~hit).sum()), 3))
    pts, pd = T.fd_points(p.cpu().numpy(), dd.cpu().numpy())
    assert torch.equal(got["normal"][torch.from_numpy(hit)], torch.from_numpy(T.fd_normals(field(pts, pd), p.cpu().numpy())))
    assert torch.equal(got["normal"][torch.from_numpy(~hit)], torch.zeros(int((~hit).sum()), 3))
    # default level: the shared table's
    dflt = render.render_surface(camera=cam, **BUNNY_IMAGE)
    assert torch.equal(dflt["depth"], render.render_surface(camera=cam, level=0.0275, **BUNNY_IMAGE)["depth"])


def test_render_surface_equals_twin_neus():
    from neddf_b200.neus import unit_normals
    from tests.test_neus_gpu import build
    from tests.test_neus_oracle import NeusCase
    render, cam = build(NeusCase("relu"))
    net = render.get_network()
    image = dict(width=64, height=48, downsampling=1)
    d, o = image_rays(render, cam, **image)
    # a level the seeded network's SDF crosses along these rays: a low quantile of its values over the depth range
    ts = np.linspace(render.dist_near, render.dist_far, 16, dtype=np.float32)
    samples = net_field(net, "sdf")((o[:, None] + ts[None, :, None] * d[:, None]).reshape(-1, 3).astype(np.float32),
                                    np.repeat(d, 16, 0))
    level = float(np.quantile(samples, 0.2))
    net, img, got, hit, p, dd, field = check_against_twin(render, cam, "sdf", level, image)
    from neddf_b200 import Sampling
    with torch.no_grad():
        out = net.forward(Sampling(p[None], dd[None], p[None]), with_normal=True)
    assert torch.equal(got["color"][torch.from_numpy(hit)], out["color"].reshape(-1, 3).cpu())
    assert torch.equal(got["normal"][torch.from_numpy(hit)], unit_normals(out["normal"].reshape(-1, 3)).cpu())


# ---------------------------------------------------------------------------------------------- against oracle --
WITNESS = 2e-5  # decision margin below which an engine's fp32 field may legitimately take the other branch


@pytest.mark.parametrize("engine", ["fp32", "tc", "tc2"])
@pytest.mark.parametrize("level", [None, 0.07])
def test_bunny_matches_oracle(engine, level):
    res, d, o, level, near, far, field = bunny_reference(level)
    render, cam = bunny(engine)
    got = {k: v.cpu().numpy() for k, v in flat(render.render_surface(camera=cam, level=level, **BUNNY_IMAGE)).items()}
    ref_hit = res["state"] == T.HIT
    # a hit decides 0 <= g < EPS, so every hit is within EPS / 2 of a decision: the witness exempts the mask only, and
    # only where the margin is below the engines' field error (measured on an H100: depth |dz| <= 6.4e-6 on tc / tc2)
    clear = (res["margin"] >= WITNESS) & (res["steps"] < 128 - T.BISECTIONS - 1)
    flips = got["hit"] != ref_hit
    both = got["hit"] & ref_hit
    dz = np.abs(got["depth"].astype(np.float64) - res["t"])[both]
    print(f"\n[surface-oracle] engine={engine} level={level}: hits {int(got['hit'].sum())}/{int(ref_hit.sum())}, "
          f"flips {int(flips.sum())} ({int((flips & clear).sum())} clear), exempt {int((~clear).sum())}, "
          f"max |dz| {float(dz.max()) if both.any() else 0.0:.3e}")
    assert not (flips & clear).any()
    assert ref_hit.sum() >= (3 if level < 0.05 else 100)
    assert float(dz.max()) <= 1e-4


@pytest.mark.parametrize("engine", ["fp32", "tc"])
def test_neddf_normals_match_oracle_gradient(engine):
    from oracle import neddf_oracle as orc
    render, cam = bunny(engine)
    img = flat(render.render_surface(camera=cam, level=0.07, **BUNNY_IMAGE))
    d, o = image_rays(render, cam, **BUNNY_IMAGE)
    hit = img["hit"].cpu().numpy()
    p = torch.from_numpy(T.points(o[hit], d[hit], img["depth"].cpu().numpy()[hit])).double()[None].requires_grad_(True)
    c = Case("bunny")
    P = {k: v.double() for k, v in c.p_fine.items()}
    dist = orc.field_forward(P, c.fc, c.st, p, torch.from_numpy(d[hit]).double()[None], torch.zeros_like(p))["distance"]
    g = torch.autograd.grad(dist.sum(), p)[0][0]
    g = g / g.norm(dim=1, keepdim=True)
    cos = (img["normal"].cpu().double()[torch.from_numpy(hit)] * g).sum(1).clamp(-1, 1)
    ang = torch.rad2deg(torch.acos(cos)).numpy()
    print(f"\n[surface-normals] engine={engine}: {hit.sum()} hits, angle to the fp64 gradient median {np.median(ang):.4f} "
          f"max {ang.max():.4f} deg")
    # measured on an H100: median 0.026 / 0.031 deg, max 0.21 / 0.18 deg (fp32 / tc); bound 0.5 deg
    assert ang.max() < 0.5


# ------------------------------------------------------------------------------------------------ against mesh --
def ray_mesh(d, o, v, f, chunk=16):
    """First-hit t of rays against a triangle mesh (Moller-Trumbore, float64, vectorised; inf on a miss)."""
    v = v.astype(np.float64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    e1, e2 = b - a, c - a
    out = np.full(len(d), np.inf)
    for i in range(0, len(d), chunk):
        dd, oo = d[i:i + chunk, None].astype(np.float64), o[i:i + chunk, None].astype(np.float64)
        pv = np.cross(dd, e2[None])
        det = (e1[None] * pv).sum(-1)
        ok = np.abs(det) > 1e-12
        inv = np.where(ok, 1.0 / np.where(ok, det, 1.0), 0.0)
        tv = oo - a[None]
        u = (tv * pv).sum(-1) * inv
        qv = np.cross(tv, e1[None])
        w = (dd * qv).sum(-1) * inv
        t = (e2[None] * qv).sum(-1) * inv
        good = ok & (u >= 0) & (w >= 0) & (u + w <= 1) & (t > 0)
        out[i:i + chunk] = np.where(good, t, np.inf).min(1)
    return out


def test_bunny_surface_matches_extracted_mesh():
    render, cam = bunny("fp32")
    net = render.get_network()
    res, r = 256, 1.1
    v, f = net.extract_mesh("distance", 0.0275, cube_range=r, cube_resolution=res)
    image = dict(width=480, height=480, downsampling=10)
    img = render.render_surface(camera=cam, level=0.0275, **image)
    d, o = image_rays(render, cam, **image)
    tm = ray_mesh(d, o, v.cpu().numpy(), f.cpu().numpy())
    mesh_hit = np.isfinite(tm) & (tm >= render.dist_near) & (tm <= render.dist_far)
    hit = img["hit"].cpu().numpy().reshape(-1)
    h, w = img["hit"].shape[:2]

    def edge(m):
        m = m.reshape(h, w)
        e = np.zeros_like(m)
        e[1:] |= m[1:] != m[:-1]
        e[:-1] |= m[1:] != m[:-1]
        e[:, 1:] |= m[:, 1:] != m[:, :-1]
        e[:, :-1] |= m[:, 1:] != m[:, :-1]
        return e.reshape(-1)

    sil = edge(hit) | edge(mesh_hit)
    both = hit & mesh_hit
    dz = np.abs(img["depth"].cpu().numpy().reshape(-1)[both] - tm[both])
    voxel = 2 * r / (res - 1)
    flips = (hit != mesh_hit) & ~sil
    print(f"\n[surface-mesh] {len(f)} faces, traced hits {hit.sum()}, mesh hits {mesh_hit.sum()}, both {both.sum()}, "
          f"non-silhouette flips {flips.sum()} of {(~sil).sum()}, depth |dz| max {dz.max() if both.any() else 0:.4e} "
          f"median {np.median(dz) if both.any() else 0:.4e} (voxel {voxel:.4e})")
    # measured on an H100: 16 pixels hit on both sides, |dz| max 4.2e-3 (0.49 voxel), 0 flips of 2267 pixels
    assert both.sum() > 0
    assert dz.max() <= 2 * voxel
    assert flips.sum() <= 2


# ------------------------------------------------------------------------------------------------- edge cases --
def test_camera_looking_away_misses_everything():
    import neddf_b200
    c = Case("bunny")
    render, _ = bunny("auto")
    R = c.z["cam_R"] @ np.diag([-1.0, 1.0, -1.0]).astype(np.float32)  # half a turn about the camera's up axis
    cam = neddf_b200.Camera.from_matrix(neddf_b200.PinholeCalib(c.z["cam_calib"]), R, c.z["cam_T"]).to(DEV)
    cam.update_transform()
    # away from the bunny the learned distance is unconstrained and dips below the default level in places; below
    # d_near (the distance's lower bound, softplus + d_near) no ray can hit, so every ray must end as a miss
    img = render.render_surface(camera=cam, level=0.5 * render.get_network().d_near, **BUNNY_IMAGE)
    assert not bool(img["hit"].any()) and bool((img["depth"] == render.dist_far).all())
    assert bool((img["normal"] == 0).all()) and bool((img["color"] == 0).all())


def test_one_pixel_and_downsampling():
    render, cam = bunny("auto")
    one = render.render_surface(1, 1, cam)
    assert one["depth"].shape == (1, 1, 1) and one["color"].shape == (1, 1, 3)
    full = render.render_surface(480, 480, cam, downsampling=10, level=0.07)
    half = render.render_surface(480, 480, cam, downsampling=20, level=0.07)
    assert bool(half["hit"].any())
    for k in full:
        assert torch.equal(half[k], full[k][::2, ::2]), k


def test_auto_engine_leaves_fp16_range_gracefully():
    import warnings
    render, cam = bunny("auto")
    with torch.no_grad():
        render.network_fine.layers_col[0].weight.mul_(1e5)  # colour trunk only: the distance field stays as it is
    assert render.network_fine.resolved_engine() == "tc"
    with pytest.warns(RuntimeWarning, match="fp16 range"):
        out = render.render_surface(camera=cam, level=0.07, **BUNNY_IMAGE)
    assert render.network_fine.resolved_engine() == "fp32"
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)  # no second detour
        again = render.render_surface(camera=cam, level=0.07, **BUNNY_IMAGE)
    render.set_engine("fp32")
    ref = render.render_surface(camera=cam, level=0.07, **BUNNY_IMAGE)
    for k in ref:
        assert torch.equal(out[k], ref[k]) and torch.equal(again[k], ref[k]), k
    assert bool(ref["hit"].any()) and float(ref["color"].abs().max()) > 1e3


# ------------------------------------------------------------------------------------------------------- CLI --
def test_surface_command_writes_pngs(tmp_path):
    import cv2
    import yaml
    c = Case("bunny")
    run = tmp_path / "bunny_run"
    (run / ".hydra").mkdir(parents=True)
    (run / "models").mkdir()
    with open(run / ".hydra" / "config.yaml", "w") as fh:
        yaml.safe_dump({"render": c.render_cfg, "network": c.net_cfg}, fh)
    torch.save(c.state_dict(), run / "models" / "model_02000.pth")
    env = dict(os.environ)
    env["PYTHONPATH"] = REPO + os.pathsep + env.get("PYTHONPATH", "")
    r = subprocess.run([sys.executable, "-m", "neddf_b200.surface", str(run), "--views", "2", "--size", "40"], cwd=REPO,
                       env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout
    for k in range(2):
        for name, shape in (("color", (40, 40, 3)), ("normal", (40, 40, 3)), ("depth", (40, 40))):
            a = cv2.imread(str(run / "surface" / f"{k:03}_{name}.png"), cv2.IMREAD_UNCHANGED)
            assert a is not None and a.shape == shape and a.dtype == np.uint8, (k, name)
    depth = cv2.imread(str(run / "surface" / "000_depth.png"), cv2.IMREAD_UNCHANGED)
    assert (depth == 255).any()  # misses are white
