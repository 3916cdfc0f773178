"""CPU: the sphere-tracing twin (tests/trace_reference.py) on analytic fields with known intersections and on the
oracle's bunny NeDDF (the CPU reference of tests/test_surface_gpu.py), and the host logic of render_surface that runs
before any device work."""
import functools

import numpy as np
import pytest
import torch

from tests import trace_reference as T

NEAR, FAR = 1.0, 8.0


def fan(n, spread, z0=-4.0):
    """Rays from (0, 0, z0) toward (x, y, 0) for x, y on an n x n grid in [-spread, spread]."""
    xs = np.linspace(-spread, spread, n)
    tgt = np.stack(np.meshgrid(xs, xs, indexing="ij"), -1).reshape(-1, 2)
    d = np.concatenate([tgt, np.full((len(tgt), 1), -z0)], 1)
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    o = np.tile(np.array([0.0, 0.0, z0], np.float32), (len(d), 1))
    return d, o


def sphere_hits(d, o, r):
    """Closed-form first intersection with |p| = r (float64), NaN for a miss."""
    d64, o64 = d.astype(np.float64), o.astype(np.float64)
    b = (d64 * o64).sum(1)
    disc = b * b - ((o64 * o64).sum(1) - r * r)
    return np.where(disc >= 0, -b - np.sqrt(np.maximum(disc, 0)), np.nan)


def test_sphere_hits_within_eps():
    d, o = fan(9, 0.5)
    res = T.trace(T.sphere_sdf((0, 0, 0), 1.0), d, o, NEAR, FAR, 0.0, 128)
    ts = sphere_hits(d, o, 1.0)
    assert np.isfinite(ts).all()
    assert (res["state"] == T.HIT).all()
    # g(t) in [0, EPS): t lies before the surface, by at most EPS / cos(incidence)
    cos_inc = np.abs((d.astype(np.float64) * (o + ts[:, None] * d)).sum(1))  # |d . n| at the hit, r = 1
    gap = ts - res["t"].astype(np.float64)
    assert (gap >= -1e-6).all(), gap.min()
    assert (gap <= float(T.EPS) / cos_inc + 1e-6).all(), (gap / (float(T.EPS) / cos_inc)).max()
    assert (res["steps"] < 40).all() and res["live_counts"][-1] == 0


def test_rays_that_miss_end_at_far():
    d, o = fan(7, 3.0)
    ts = sphere_hits(d, o, 1.0)
    res = T.trace(T.sphere_sdf((0, 0, 0), 1.0), d, o, NEAR, FAR, 0.0, 128)
    miss = np.isnan(ts)
    assert miss.sum() > 10 and (~miss).sum() > 0
    assert (res["state"][miss] == T.MISS).all() and (res["t"][miss] == np.float32(FAR)).all()
    assert (res["state"][~miss] == T.HIT).all()


def test_grazing_plane_ends_at_max_steps():
    """A ray at 0.5 degrees to the plane z = 0 approaches it by a factor (1 - sin 0.5deg) per step: far more than
    max_steps steps to reach EPS, and far beyond the horizon only after ~100 units."""
    a = np.radians(0.5)
    d = np.array([[np.cos(a), 0.0, -np.sin(a)]], np.float32)
    o = np.array([[0.0, 0.0, 1.0]], np.float32)
    res = T.trace(T.plane_sdf((0, 0, 1), 0.0), d, o, 0.0, 1000.0, 0.0, 64)
    assert res["state"][0] == T.MISS and res["steps"][0] == 64 and res["t"][0] == np.float32(1000.0)
    res = T.trace(T.plane_sdf((0, 0, 1), 0.0), d, o, 0.0, 1000.0, 0.0, 4000)
    assert res["state"][0] == T.HIT and 64 < res["steps"][0] < 4000


def test_doubled_sdf_overshoots_and_bisects():
    d, o = fan(9, 0.5)
    field = T.sphere_sdf((0, 0, 0), 1.0, scale=2.0)
    # from t = 2.5 a 2 x SDF step lands as far behind the surface as it started in front of it (not yet through the
    # sphere): every ray bisects, and its hit is the near end of an 8-fold halved bracket, on the camera's side
    res = T.trace(field, d, o, 2.5, FAR, 0.0, 128)
    assert (res["state"] == T.HIT).all()
    bisected = res["hi"] > res["lo"]
    g_hit = field(T.points(o, d, res["t"]), d)
    assert (g_hit >= 0).all()
    ts = sphere_hits(d, o, 1.0)
    width = (res["hi"] - res["lo"]).astype(np.float64)
    assert bisected.all() and (res["t"] == res["lo"]).all()
    gap = ts - res["t"].astype(np.float64)
    assert (gap >= -1e-6).all() and (gap <= width + 1e-6).all()


def test_max_steps_cuts_a_bisection():
    d, o = fan(3, 0.5)
    field = T.sphere_sdf((0, 0, 0), 1.0, scale=2.0)
    full = T.trace(field, d, o, 2.5, FAR, 0.0, 128)
    assert (full["state"] == T.HIT).all()
    cut = T.trace(field, d, o, 2.5, FAR, 0.0, int(full["steps"].min()) - 1)
    assert (cut["state"] == T.MISS).all() and (cut["t"] == np.float32(FAR)).all()


def test_start_inside_is_a_miss():
    d, o = fan(3, 0.2)
    res = T.trace(T.sphere_sdf((0, 0, -4), 1.0), d, o, 0.5, FAR, 0.0, 128)
    assert (res["state"] == T.MISS).all() and (res["steps"] == 1).all()


def test_fd_normals_of_a_sphere():
    d, o = fan(9, 0.5)
    field = T.sphere_sdf((0, 0, 0), 1.0)
    res = T.trace(field, d, o, NEAR, FAR, 0.0, 128)
    p = T.points(o, d, res["t"])
    pts, pd = T.fd_points(p, d)
    n = T.fd_normals(field(pts, pd), p)
    radial = p / np.linalg.norm(p.astype(np.float64), axis=1, keepdims=True)
    assert np.abs(np.linalg.norm(n.astype(np.float64), axis=1) - 1).max() < 1e-6
    assert (n * radial).sum(1).min() > 0.999


# ------------------------------------------------------------------------------------------------------ bunny --
BUNNY_IMAGE = dict(width=480, height=480, downsampling=20)  # the case_bunny camera (cx = cy = 250), 24 x 24 pixels


@functools.lru_cache(maxsize=4)
def bunny_reference(level=None, max_steps: int = 128):
    """The twin on the oracle's bunny NeDDF (float64 field at the twin's fp32 points), over the 24 x 24 image of the
    case_bunny camera, rays from the oracle's make_rays; ``level=None``: the NeDDF default.
    -> (trace result, ray_dir, ray_orig, level, near, far, field)."""
    from neddf_b200.network import LEVEL_DEFAULTS
    from oracle import neddf_oracle as orc
    from tests.helpers import Case
    c = Case("bunny")
    P = {k: v.double() for k, v in c.p_fine.items()}
    uv = orc.image_uv(**BUNNY_IMAGE)
    d, o = orc.make_rays(uv, c.cam)
    d, o = d.numpy().astype(np.float32), o.contiguous().numpy().astype(np.float32)

    def field(p, dirs):
        pt = torch.from_numpy(p).double()[None]
        with torch.no_grad():
            out = orc.field_forward(P, c.fc, c.st, pt, torch.from_numpy(dirs).double()[None], torch.zeros_like(pt))
        return out["distance"].reshape(-1).numpy().astype(np.float32)

    level = LEVEL_DEFAULTS["NeDDF"][1] if level is None else level
    res = T.trace(field, d, o, c.rc.dist_near, c.rc.dist_far, level, max_steps)
    return res, d, o, level, c.rc.dist_near, c.rc.dist_far, field


@pytest.mark.parametrize("level,min_hits", [(None, 3), (0.07, 100)])
def test_bunny_reference_is_a_surface(level, min_hits):
    """The smoke checkpoint is briefly trained: at the default level its distance field reaches the level set on only a
    few of these pixels (the central ray's distance bottoms out at 0.049), at 0.07 on a quarter of them."""
    res, d, o, level, near, far, field = bunny_reference(level)
    hit = res["state"] == T.HIT
    assert min_hits <= hit.sum() < 0.9 * hit.size, hit.sum()
    assert set(np.unique(res["state"])) <= {T.HIT, T.MISS}
    g = field(T.points(o[hit], d[hit], res["t"][hit]), d[hit]) - np.float32(level)
    assert (g >= 0).all() and (res["t"][hit] > near).all() and (res["t"][~hit] == np.float32(far)).all()
    assert res["steps"].max() <= 128


# ----------------------------------------------------------------------------------------------- host logic --
def cpu_render(net_cfg, render_cfg=None):
    import neddf_b200
    return neddf_b200.NeRFRender(network_config=dict(net_cfg), **(render_cfg or {}))


def test_nerf_has_no_surface_to_trace():
    from tests.test_nerf_oracle import NerfCase
    r = cpu_render(NerfCase("relu").net_cfg)
    with pytest.raises(ValueError, match="no distance field"):
        r.render_surface(8, 8, camera=None)
    with pytest.raises(ValueError, match="no distance field"):
        r.get_network().surface_level(0.5)


def test_levels_come_from_the_shared_table(monkeypatch):
    import neddf_b200
    from neddf_b200 import network
    assert neddf_b200.NeDDF().surface_level() == network.LEVEL_DEFAULTS["NeDDF"][1] == 0.0275
    assert neddf_b200.NeuS().surface_level() == network.LEVEL_DEFAULTS["NeuS"][1] == 0.0
    assert neddf_b200.NeDDF().surface_level(0.1) == 0.1
    monkeypatch.setitem(network.LEVEL_DEFAULTS, "NeDDF", ("distance", 0.05))
    assert neddf_b200.NeDDF().surface_level() == 0.05
    with pytest.raises(ValueError):
        neddf_b200.NeDDF().surface_level(float("nan"))


@pytest.mark.parametrize("kw", [dict(max_steps=0), dict(max_steps=1.5), dict(max_steps=True), dict(width=0),
                                dict(height=-1), dict(downsampling=0), dict(width=3, downsampling=4)])
def test_bad_arguments_raise_before_any_device_work(kw):
    from tests.helpers import Case
    r = cpu_render(Case("bunny").net_cfg)
    args = dict(width=8, height=8, camera=None)
    args.update(kw)
    with pytest.raises(ValueError):
        r.render_surface(**args)


def test_cpu_module_is_refused():
    from tests.helpers import Case
    r = cpu_render(Case("bunny").net_cfg)
    with pytest.raises(RuntimeError, match="CUDA"):
        r.render_surface(8, 8, camera=None)
