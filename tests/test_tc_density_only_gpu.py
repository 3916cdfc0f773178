"""Density-only launches: a field launch with no colour, penalty or training output runs the tensor-core kernel's
distance trunk and distance / aux head alone (what an image's coarse pass needs: its weights depend on density only).
Checked at tile counts that are not a multiple of 2 or 4 (pairs, colour groups): distance, density and aux_grad
bit-identical to an images-only launch that also computes colour, nothing written past the requested samples, and
images bit-identical with the coarse colour skipped and computed."""
import ctypes as C
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests.helpers import Case  # noqa: E402

pytestmark = pytest.mark.gpu

ENGINES = ("tc", "tc2")
# samples = 32 x tiles + 17: 1, 3 and 5 tiles, and an odd tile count beyond 6 tiles per SM ("many")
COUNTS = (17, 81, 145, "many")
PAD = 100  # output elements past the requested samples, pre-filled with NaN
KEYS = ("distance", "density", "aux_grad")


def _count(n):
    if n != "many":
        return n
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    return 32 * (6 * sm + 2) + 17


def _setup(engine):
    import tests.gpu_util as G
    c = Case("default")
    render = G.build_render(c, engine)
    return G, c, render, render.network_fine


@pytest.mark.parametrize("n", COUNTS)
@pytest.mark.parametrize("engine", ENGINES)
def test_point_entry_density_only(engine, n):
    from neddf_b200 import _lib as L
    G, c, render, net = _setup(engine)
    n = _count(n)
    g = torch.Generator().manual_seed(n)
    pos = (torch.rand(n, 3, generator=g) - 0.5) * 2.0
    dd = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    var = torch.rand(n, 3, generator=g) * 1e-3
    p3, d3, v3 = (t.to(G.DEV).contiguous() for t in (pos, dd, var))
    h, st = net._field(G.DEV), net._state_struct()
    sentinel = -1234.5

    def run(with_color, flags=L.OUT_EVAL):
        o = {k: torch.full((n + PAD,), float("nan"), device=G.DEV) for k in KEYS}
        o["color"] = torch.full((n + PAD, 3), sentinel, device=G.DEV)
        with torch.no_grad():
            L.check(L.lib().neddf_field_forward(
                h, C.byref(st), L.ptr(p3), L.ptr(d3), L.ptr(v3), n, L.ptr(o["distance"]), L.ptr(o["density"]),
                L.ptr(o["color"]) if with_color else None, None, L.ptr(o["aux_grad"]), flags, net._engine_id(),
                L.stream_ptr(G.DEV)), "field_forward")
        torch.cuda.synchronize()
        return o

    # the density-only path does not depend on the flags: an OUT_FULL launch with no colour or penalty takes it too
    dens_only, with_col, dens_only2, full_flags = run(False), run(True), run(False), run(False, L.OUT_FULL)
    net.check_engine_status()
    for k in KEYS:
        assert torch.equal(dens_only[k][:n], with_col[k][:n]), k
        assert torch.equal(dens_only[k][:n], dens_only2[k][:n]), k
        assert torch.equal(dens_only[k][:n], full_flags[k][:n]), k
        for o in (dens_only, full_flags):
            assert torch.isnan(o[k][n:]).all(), k
        assert torch.isfinite(dens_only[k][:n]).all(), k
    # the colour buffer was never handed to the kernel, and nothing reached it
    assert (dens_only["color"] == sentinel).all() and (full_flags["color"] == sentinel).all()
    assert (with_col["color"][n:] == sentinel).all() and torch.isfinite(with_col["color"][:n]).all()


@pytest.mark.parametrize("n", COUNTS)
@pytest.mark.parametrize("engine", ENGINES)
def test_ray_entry_density_only(engine, n):
    G, c, render, net = _setup(engine)
    n = max(_count(n), 2)
    g = torch.Generator().manual_seed(n)
    n_edges = 9
    n_rays = (n + n_edges - 1) // n_edges
    d = torch.nn.functional.normalize(torch.randn(n_rays, 3, generator=g) + torch.tensor([0.0, 0.0, -3.0]), dim=-1)
    o = torch.randn(n_rays, 3, generator=g) * 0.1 + torch.tensor([0.0, 0.0, 2.5])
    dists = torch.sort(1.0 + 3.0 * torch.rand(n_rays, n_edges, generator=g), dim=-1).values
    args = (d.to(G.DEV), o.to(G.DEV), dists.to(G.DEV), c.rc.sampling_type, render._ray_radius)
    with torch.no_grad():
        dens_only = net.forward_rays(*args, need_penalty=False, need_aux=True, need_color=False)
        with_col = net.forward_rays(*args, need_penalty=False, need_aux=True, need_color=True)
    net.check_engine_status()
    assert "color" not in dens_only and "color" in with_col
    for k in KEYS:
        assert torch.equal(dens_only[k], with_col[k]), k


@pytest.mark.parametrize("engine", ("fp32", "tc", "tc2"))
def test_render_pixels_skips_coarse_colour_bit_identically(engine):
    """An image's coarse pass runs density-only unless a *_coarse target is asked for; colour and depth of the
    image are the same bit for bit either way."""
    import tests.gpu_util as G
    c = Case("bunny")
    render, cam = G.build_render(c, engine), G.build_camera(c)
    W, H = 64, 48
    count = W * H - 5  # a ray count that is no multiple of a tile
    g = torch.Generator(device=G.DEV).manual_seed(7)
    u = (torch.rand(count, render.sample_coarse + 1, generator=g, device=G.DEV),
         torch.rand(count, render.sample_fine + 1, generator=g, device=G.DEV))
    skipped = render.render_pixels(W, H, cam, ["color", "depth"], 1, 3, count, uniforms=u)
    forced = render.render_pixels(W, H, cam, ["color", "depth", "color_coarse", "depth_coarse"], 1, 3, count, uniforms=u)
    render.check_status()
    for k in ("color", "depth"):
        assert torch.equal(skipped[k], forced[k]), k
        assert torch.isfinite(skipped[k]).all(), k
    assert torch.isfinite(forced["color_coarse"]).all()


def test_composite_without_colour():
    """integrate_volume_render(colors=None): weight, depth and transmittance as with colours, and no "color"."""
    import tests.gpu_util as G
    c = Case("default")
    render = G.build_render(c, "fp32")
    g = torch.Generator().manual_seed(3)
    B, E = 37, 65
    dists = torch.sort(2.0 + 4.0 * torch.rand(B, E, generator=g), dim=-1).values.to(G.DEV)
    dens = (torch.rand(B, E, generator=g) * 5.0).to(G.DEV)
    col = torch.rand(B, E, 3, generator=g).to(G.DEV)
    with torch.no_grad():
        a = render.integrate_volume_render(dists, dens, None)
        b = render.integrate_volume_render(dists, dens, col)
    assert "color" not in a
    for k in ("weight", "depth", "transmittance"):
        assert torch.equal(a[k], b[k]), k
