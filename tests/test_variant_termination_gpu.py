"""Early ray termination for the NeRF and NeuS networks on the GPU (neddf_nerf_forward_rays_segment,
neddf_neus_forward_rays_segment behind NeRF / NeuS.forward_rays_segment, driven by NeRFRender._fine_pass_terminated).

- With eps below every ray's final transmittance no ray stops: the image is bitwise the render with termination off,
  for 2, 3, 5 and E segments, and every nominal evaluation runs.
- With an eps at which rays stop, the device's executed count equals the count predicted on the host from the full
  render's densities, and the image stays within the stated error bound.
- Direct ABI calls at the structural extremes of tests/nerf_neus_configs.py equal the whole-row forward on the entries
  they evaluate and write nothing else; argument errors and autograd are refused.
- render_image_sharded over two gloo ranks on one device equals the single-GPU terminated render."""
import ctypes as C
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import nerf_neus_configs as ncfg
from tests.test_nerf_oracle import NerfCase
from tests.test_neus_oracle import NeusCase

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
WIDTH = HEIGHT = 800  # the goldens' 800 x 800 camera, downsampled to 40 x 40 pixels
DS = 20
KEYS = ["color", "depth", "transmittance"]


def _camera(z):
    import neddf_b200
    cam = neddf_b200.Camera.from_matrix(neddf_b200.PinholeCalib(z["cam_calib"]), z["cam_R"], z["cam_T"]).to(DEV)
    cam.update_transform()
    return cam


def _golden(variant: str, name: str, sampling=None):
    from tests.test_nerf_gpu import build as build_nerf
    from tests.test_neus_gpu import build as build_neus
    render, cam = build_nerf(NerfCase(name)) if variant == "nerf" else build_neus(NeusCase(name))
    if sampling is not None:
        render.sampling_type = sampling
    return render, cam


def _sharp_neus():
    """S5_sharp (init_variance 2, an sdf running from tanhExp's floor to above 5 across the unit cube) as the one
    network of a NeRFRender, seen by the NeuS ReLU golden's camera: rays that cross its zero set turn opaque."""
    import neddf_b200
    c = NeusCase("relu")
    cfg = dict(c.render_cfg, use_coarse_network=False)
    render = neddf_b200.NeRFRender(network_config={"_target_": "neddf.network.NeuS", **ncfg.kwargs("S5_sharp")}, **cfg)
    render.network_fine.load_state_dict(ncfg.state_dict("S5_sharp"))
    render.to(DEV)
    render.set_iter(-1)
    return render, _camera(c.z)


def _uniforms(render, seed=11):
    n_pix = (WIDTH // DS) * (HEIGHT // DS)
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n_pix, render.sample_coarse + 1, generator=g).to(DEV),
            torch.rand(n_pix, render.sample_fine + 1, generator=g).to(DEV))


def _image(render, cam, u, eps=0.0, segments=4):
    render.transmittance_eps, render.termination_segments = float(eps), int(segments)
    out = render.render_image(WIDTH, HEIGHT, cam, KEYS, DS, uniforms=u)
    return out, render.termination_stats()


GOLDENS = [("nerf", "relu", None), ("nerf", "relu", "point"), ("nerf", "tanhexp", None), ("nerf", "tanhexp", "cone"),
           ("neus", "relu", None), ("neus", "tanhexp", None)]


@pytest.mark.parametrize("variant, name, sampling", GOLDENS,
                         ids=["nerf-relu-shared-cone", "nerf-relu-shared-point", "nerf-tanhexp-separate-point",
                              "nerf-tanhexp-separate-cone", "neus-relu", "neus-tanhexp"])
def test_termination_is_invisible_when_no_ray_stops(variant, name, sampling):
    """eps at half the smallest final transmittance: no ray can stop, so the image is the render with termination off
    under torch.equal for 2, 3, 5 and E segments, and every nominal evaluation is executed."""
    render, cam = _golden(variant, name, sampling)
    u = _uniforms(render)
    base, st = _image(render, cam, u)
    assert st == {"executed": 0, "nominal": 0}  # eps = 0: the reference's fine pass, no counters
    t_min = float(base["transmittance"].min())
    assert t_min > 0.0
    E = render.sample_coarse + render.sample_fine + 2
    n_pix = u[0].shape[0]
    for segments in (2, 3, 5, E):
        out, st = _image(render, cam, u, 0.5 * t_min, segments)
        assert st["executed"] == st["nominal"] == n_pix * E, (segments, st)
        for k in KEYS:
            assert torch.equal(out[k], base[k]), (segments, k, float((out[k] - base[k]).abs().max()))
    render.check_status()


def _capture_fine_pass(render, cam, u):
    """The eps = 0 image and its fine pass's (dists, density, colour), recorded from network_fine.forward_rays (the
    coarse pass has sample_coarse + 1 edges per ray, the fine pass sample_coarse + sample_fine + 2)."""
    net = render.network_fine
    E = render.sample_coarse + render.sample_fine + 2
    rec = []
    inner = net.forward_rays

    def recording(ray_dir, ray_orig, dists, *a, **kw):
        out = inner(ray_dir, ray_orig, dists, *a, **kw)
        if dists.shape[1] == E:
            rec.append((dists.clone(), out["density"].clone(), out["color"].clone()))
        return out

    net.forward_rays = recording
    try:
        base, _ = _image(render, cam, u)
    finally:
        del net.forward_rays
    assert len(rec) == 1  # one chunk
    return base, rec[0]


def _segment_ends(dists, density, K):
    """Each ray's transmittance at the end of each of the renderer's K segments, in fp64 from the fp32 densities and
    the fp32 interval lengths neddf_terminate_rays uses: T *= 1 - o_j + 1e-7, o_j = 1 - exp(-density_j delta_j)."""
    B, E = dists.shape
    delta = (dists[:, 1:] - dists[:, :-1]).double().cpu()
    fac = 1.0 - (1.0 - torch.exp(-density[:, :-1].double().cpu() * delta)) + 1e-7
    bounds = [round(k * E / K) for k in range(K + 1)]
    T, ends = torch.ones(B, dtype=torch.float64), []
    for k in range(K):
        T = T * fac[:, bounds[k]:min(bounds[k + 1], E - 1)].prod(1)
        ends.append(T.clone())
    return bounds, ends


def _choose_eps(ends):
    """An eps at which some ray stops before the last segment, as far (relatively) as the data allow from every
    segment-end transmittance: the geometric middle of the widest gap above a non-final transmittance below 1e-3,
    1e-2, 0.1 or 0.5 (the first of these with one)."""
    early = torch.cat(ends[:-1])
    every = torch.sort(torch.cat(ends)).values
    for target in (1e-3, 1e-2, 0.1, 0.5):
        cand = early[(early <= target) & (early >= target / 10)]
        if cand.numel() == 0:
            cand = early[early <= target]
        if cand.numel() == 0:
            continue
        best, eps = 0.0, None
        for lo in torch.unique(cand)[-64:].tolist():
            hi = float(every[every > lo][0]) if bool((every > lo).any()) else 2 * lo + 1e-30
            ratio = hi / max(lo, 1e-300)
            if ratio > best:
                best, eps = ratio, (lo * hi) ** 0.5 if lo > 0 else hi / 2
        return eps
    pytest.fail("no ray's transmittance falls below 0.5 before its last segment")


@pytest.mark.parametrize("variant, name", [("nerf", "relu"), ("nerf", "tanhexp"), ("neus", "sharp")])
def test_executed_count_and_error_bound_when_rays_stop(variant, name):
    """eps chosen where rays stop (at least 1e-6 relative from every segment-end transmittance of the full render):
    the device's executed count equals the host's fp64 prediction exactly, and colour, depth and transmittance stay
    within |dc| <= eps max|c|, |d depth| <= eps max_dist, |dT| <= eps of the full render."""
    render, cam = _sharp_neus() if name == "sharp" else _golden(variant, name)
    u = _uniforms(render)
    base, (dists, density, colour) = _capture_fine_pass(render, cam, u)
    B, E = dists.shape
    K = 4
    bounds, ends = _segment_ends(dists, density, K)
    eps = _choose_eps(ends)
    margin = min(float(((T - eps).abs() / eps).min()) for T in ends)
    assert margin >= 1e-6, margin
    live, expect = torch.ones(B, dtype=torch.bool), 0
    for k in range(K):
        expect += int(live.sum()) * (bounds[k + 1] - bounds[k])
        live &= ends[k] > eps
    assert expect < B * E  # some ray stopped before its last segment
    out, st = _image(render, cam, u, eps, K)
    assert st == {"executed": expect, "nominal": B * E}, (st, expect, B * E, eps, margin)
    # the bound, with room for fp32 rounding: a stopped ray's transmittance keeps the closing factors (1 + 1e-7)
    slack = 1 + 1e-4
    c_max = float(colour.abs().max())
    assert float((out["color"] - base["color"]).abs().max()) <= eps * c_max * slack + 1e-6
    assert float((out["depth"] - base["depth"]).abs().max()) <= eps * render.max_dist * slack + 1e-6
    assert float((out["transmittance"] - base["transmittance"]).abs().max()) <= eps * slack + 1e-7
    stopped = torch.zeros(B, dtype=torch.bool)
    for T in ends[:-1]:
        stopped |= T <= eps
    # rays that never stopped are the full render's, bit for bit
    flat = {k: v.reshape(B, -1).cpu() for k, v in out.items()}
    ref = {k: v.reshape(B, -1).cpu() for k, v in base.items()}
    for k in KEYS:
        assert torch.equal(flat[k][~stopped], ref[k][~stopped]), k


# ------------------------------------------------------------------------------------ direct ABI calls --

def _network(name):
    import neddf_b200
    cls = neddf_b200.NeRF if ncfg.variant(name) == "nerf" else neddf_b200.NeuS
    net = cls(**ncfg.kwargs(name))
    net.load_state_dict(ncfg.state_dict(name))
    net.set_iter(ncfg.CONFIGS[name]["iter"])
    return net.to(DEV)


def _segment_call(net, d, o, dists, e0, seg, idx, n_active, den, col, n_rays=None):
    from neddf_b200 import _lib as L
    from neddf_b200.ray import CONE_RAY_RADIUS
    lib = L.lib()
    B, E = dists.shape
    B = B if n_rays is None else n_rays
    h = net._field(DEV)
    args = (L.ptr(d), L.ptr(o), L.ptr(dists), B, E, L.SAMPLING_IDS["cone"], CONE_RAY_RADIUS, e0, seg, L.ptr(idx), L.ptr(n_active),
            L.ptr(den), L.ptr(col), L.stream_ptr(DEV))
    if hasattr(net, "lowpass_alpha"):
        return lib.neddf_nerf_forward_rays_segment(h, net._lowpass(), *args)
    return lib.neddf_neus_forward_rays_segment(h, *args)


@pytest.mark.parametrize("name", ["N2_max_embed", "N3_deep_fwd", "N5_eight_skips", "S2_max_embed", "S3_deepest", "S4_eight_skips"])
def test_segment_abi_at_structural_extremes(name):
    """One segment of length 1 over all 67 rays (67 samples: not a multiple of the 64-sample tile), a segment that ends
    on the closing edge over a ray list (reversed odd rays), n_active = 0, no rays at all: the evaluated entries equal
    neddf_*_forward_rays bit for bit, every other entry keeps its zero."""
    from neddf_b200.ray import CONE_RAY_RADIUS
    net = _network(name)
    d, o, dists = (t.to(DEV) for t in ncfg.rays(67, 9, ncfg.SEED[name] + 5))
    B, E = dists.shape
    with torch.no_grad():
        full = net.forward_rays(d, o, dists, "cone", CONE_RAY_RADIUS)
    odd = torch.arange(B - 1 if B % 2 == 0 else B - 2, 0, -2, dtype=torch.int32, device=DEV)
    cases = [("one edge", 4, 1, None, None), ("closing edge", 5, 4, odd, torch.tensor([odd.numel()], dtype=torch.int32, device=DEV)),
             ("n_active 0", 0, 9, odd, torch.zeros(1, dtype=torch.int32, device=DEV))]
    for what, e0, seg, idx, n_active in cases:
        den = torch.zeros(B, E, device=DEV)
        col = torch.zeros(B, E, 3, device=DEV)
        assert _segment_call(net, d, o, dists, e0, seg, idx, n_active, den, col) == 0, what
        torch.cuda.synchronize()
        mask = torch.zeros(B, E, dtype=torch.bool, device=DEV)
        if idx is not None:
            rows = idx[:int(n_active.item())].long()
            mask[rows, e0:e0 + seg] = True
        else:
            mask[:, e0:e0 + seg] = True
        assert torch.equal(den[mask], full["density"][mask]) and torch.equal(col[mask], full["color"][mask]), what
        assert not den[~mask].any() and not col[~mask].any(), what
    den, col = torch.zeros(1, E, device=DEV), torch.zeros(1, E, 3, device=DEV)
    assert _segment_call(net, d, o, dists, 0, 2, None, None, den, col, n_rays=0) == 0  # no rays: nothing to do
    torch.cuda.synchronize()
    assert not den.any() and not col.any()


@pytest.mark.parametrize("name", ["N2_max_embed", "S2_max_embed"])
def test_segment_refusals_raise(name):
    """Argument errors of the new entry points raise RuntimeError from Python; forward_rays_segment under autograd
    raises before any launch."""
    from neddf_b200.ray import CONE_RAY_RADIUS
    net = _network(name)
    d, o, dists = (t.to(DEV) for t in ncfg.rays(5, 9, 3))
    den, col = torch.zeros(5, 9, device=DEV), torch.zeros(5, 9, 3, device=DEV)
    idx = torch.arange(5, dtype=torch.int32, device=DEV)
    cnt = torch.tensor([5], dtype=torch.int32, device=DEV)
    with torch.no_grad():
        for e0, seg, i, n, msg in ((-1, 2, None, None, "bad segment"), (0, 0, None, None, "bad segment"),
                                   (8, 2, None, None, "bad segment"), (0, 2, idx, None, "go together"),
                                   (0, 2, None, cnt, "go together")):
            with pytest.raises(RuntimeError, match=msg):
                net.forward_rays_segment(d, o, dists, "cone", CONE_RAY_RADIUS, e0, seg, i, n, den, col)
        with pytest.raises(RuntimeError, match="sampling_type"):
            _lib_call_bad_sampling(net, d, o, dists, den, col)
    assert not den.any() and not col.any()
    with pytest.raises(RuntimeError, match="no gradient"):
        net.forward_rays_segment(d, o, dists, "cone", CONE_RAY_RADIUS, 0, 2, None, None, den, col)


def _lib_call_bad_sampling(net, d, o, dists, den, col):
    from neddf_b200 import _lib as L
    lib = L.lib()
    h = net._field(DEV)
    args = (L.ptr(d), L.ptr(o), L.ptr(dists), 5, 9, 7, 0.0, 0, 2, None, None, L.ptr(den), L.ptr(col), L.stream_ptr(DEV))
    rc = lib.neddf_nerf_forward_rays_segment(h, net._lowpass(), *args) if hasattr(net, "lowpass_alpha") else \
        lib.neddf_neus_forward_rays_segment(h, *args)
    L.check(rc, "forward_rays_segment")


# ------------------------------------------------------------------------------------------ multi-GPU --

class _HostTiles:
    """A NeRFRender whose render_pixels hands its tiles to the host: gloo gathers host tensors."""

    def __init__(self, render):
        self.render = render

    def render_pixels(self, *a, **kw):
        return {k: v.cpu() for k, v in self.render.render_pixels(*a, **kw).items()}

    def __getattr__(self, k):
        return getattr(self.render, k)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _sharded_worker(rank, world, port, eps, out_path):
    from neddf_b200.dist import render_image_sharded
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        render, cam = _golden("nerf", "relu")
        u = _uniforms(render)
        render.transmittance_eps, render.termination_segments = eps, 4
        img = render_image_sharded(_HostTiles(render), WIDTH, HEIGHT, cam, KEYS, DS, uniforms=u)
        st = render.termination_stats()
        if rank == 0:
            torch.save({"img": img, "stats": st}, out_path)
    finally:
        dist.destroy_process_group()


def test_sharded_render_with_termination_equals_single_gpu(tmp_path):
    """render_image_sharded (each rank renders its slice of the pixel list through render_pixels, so it terminates
    rays like render_image) in two gloo ranks sharing cuda:0 equals the single-GPU terminated render."""
    render, cam = _golden("nerf", "relu")
    u = _uniforms(render)
    _, (dists, density, _) = _capture_fine_pass(render, cam, u)
    eps = _choose_eps(_segment_ends(dists, density, 4)[1])  # an eps at which rays stop
    ref, st = _image(render, cam, u, eps, 4)
    out_path = str(tmp_path / "rank0.pt")
    mp.spawn(_sharded_worker, args=(2, _free_port(), eps, out_path), nprocs=2, join=True)
    got = torch.load(out_path)
    assert st["executed"] < st["nominal"]  # rays do stop at this eps
    assert 0 < got["stats"]["executed"] < st["executed"]  # rank 0 ran its own slice only
    for k in KEYS:
        assert torch.equal(got["img"][k], ref[k].cpu()), k
