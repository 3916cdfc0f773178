"""Images-only launches of the tensor-core engines run the colour trunk once per group of four 32-sample
tiles.  Checked at sample counts around the tile and group edges, through the point, cone-ray and segment
entry points: bit-identical to the same samples through the full (penalty) kernel, within the parity bar
of the fp64 oracle, repeatable, and nothing written past the requested samples."""
import ctypes as C
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import neddf_oracle as orc  # noqa: E402
from tests.helpers import PARITY_TOL, Case, nerr  # noqa: E402

pytestmark = pytest.mark.gpu

ENGINES = ("tc", "tc2")
# around one tile (32) and one group (128); "many": more tiles than 4 x CTAs with a ragged last group
COUNTS = (1, 31, 32, 33, 96, 127, 128, 129, 160, "many")
PAD = 100  # output elements past the requested samples, pre-filled with NaN


def _count(n):
    if n != "many":
        return n
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    return 32 * (4 * sm + 2 * sm + 1) + 17


def _setup(engine):
    import tests.gpu_util as G
    c = Case("default")
    render = G.build_render(c, engine)
    return G, c, render, render.network_fine


def _oracle_subset(n):
    # the fp64 oracle on every sample of the small counts, and on the first and the last group of the large one
    return torch.arange(n) if n <= 160 else torch.cat([torch.arange(128), torch.arange(n - 160, n)])


@pytest.mark.parametrize("n", COUNTS)
@pytest.mark.parametrize("engine", ENGINES)
def test_point_entry(engine, n):
    from neddf_b200 import _lib as L
    G, c, render, net = _setup(engine)
    n = _count(n)
    g = torch.Generator().manual_seed(n)
    pos = (torch.rand(n, 3, generator=g) - 0.5) * 2.0
    dd = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    var = torch.rand(n, 3, generator=g) * 1e-3
    p3, d3, v3 = (t.to(G.DEV).contiguous() for t in (pos, dd, var))
    h, st = net._field(G.DEV), net._state_struct()

    def run(penalty):
        o = {k: torch.full((n + PAD,) + ((3,) if k == "color" else ()), float("nan"), device=G.DEV)
             for k in ("distance", "density", "color", "fields_penalty", "aux_grad")}
        with torch.no_grad():
            L.check(L.lib().neddf_field_forward(
                h, C.byref(st), L.ptr(p3), L.ptr(d3), L.ptr(v3), n, L.ptr(o["distance"]), L.ptr(o["density"]),
                L.ptr(o["color"]), L.ptr(o["fields_penalty"]) if penalty else None, L.ptr(o["aux_grad"]),
                L.OUT_FULL if penalty else L.OUT_EVAL, net._engine_id(), L.stream_ptr(G.DEV)), "field_forward")
        torch.cuda.synchronize()
        return o

    ev, ev2, full = run(False), run(False), run(True)
    net.check_engine_status()
    for k in ("distance", "density", "color", "aux_grad"):
        assert torch.equal(ev[k][:n], full[k][:n]), k
        assert torch.equal(ev[k][:n], ev2[k][:n]), k
        assert torch.isnan(ev[k][n:]).all(), k
    idx = _oracle_subset(n)
    ref = orc.field_forward(c.p_fine, c.fc, c.st, pos[idx][None], dd[idx][None], var[idx][None])
    for k in ("distance", "density", "color", "aux_grad"):
        assert nerr(ev[k][:n][idx.to(G.DEV)].cpu().numpy(), ref[k][0].numpy()) < PARITY_TOL, k


def _rays(n_rays, n_edges, seed):
    g = torch.Generator().manual_seed(seed)
    d = torch.nn.functional.normalize(torch.randn(n_rays, 3, generator=g) + torch.tensor([0.0, 0.0, -3.0]), dim=-1)
    o = torch.randn(n_rays, 3, generator=g) * 0.1 + torch.tensor([0.0, 0.0, 2.5])
    dists = torch.sort(1.0 + 3.0 * torch.rand(n_rays, n_edges, generator=g), dim=-1).values
    return d, o, dists


@pytest.mark.parametrize("n", COUNTS)
@pytest.mark.parametrize("engine", ENGINES)
def test_cone_ray_entry(engine, n):
    G, c, render, net = _setup(engine)
    n = max(_count(n), 2)  # one ray of n samples (a frustum needs two edges; one sample is in the point test)
    d, o, dists = _rays(1, n, n)
    args = (d.to(G.DEV), o.to(G.DEV), dists.to(G.DEV), c.rc.sampling_type, render._ray_radius)
    with torch.no_grad():
        ev = net.forward_rays(*args, need_penalty=False, need_aux=True)
        ev2 = net.forward_rays(*args, need_penalty=False, need_aux=True)
        full = net.forward_rays(*args, need_penalty=True, need_aux=True)
    net.check_engine_status()
    for k in ("distance", "density", "color", "aux_grad"):
        assert torch.equal(ev[k], full[k]), k
        assert torch.equal(ev[k], ev2[k]), k
    idx = _oracle_subset(n)
    pos, dd, var = orc.make_samples(c.rc, d, o, dists)
    pos, dd, var = (t.reshape(-1, 3)[idx][None] for t in (pos, dd.expand_as(pos), var))
    ref = orc.field_forward(c.p_fine, c.fc, c.st, pos, dd, var)
    for k in ("distance", "density", "color", "aux_grad"):
        got = ev[k].reshape(n, -1)[idx.to(G.DEV)].reshape(ref[k][0].shape)
        assert nerr(got.cpu().numpy(), ref[k][0].numpy()) < PARITY_TOL, k


@pytest.mark.parametrize("n", COUNTS)
@pytest.mark.parametrize("engine", ENGINES)
def test_segment_entry(engine, n):
    G, c, render, net = _setup(engine)
    n = _count(n)
    n_edges, edge0 = 8, 3
    seg_len = 2 if n % 2 == 0 else 1
    d, o, dists = _rays(n // seg_len, n_edges, n)
    args = (d.to(G.DEV), o.to(G.DEV), dists.to(G.DEV), c.rc.sampling_type, render._ray_radius)
    with torch.no_grad():
        full = net.forward_rays(*args, need_penalty=True, need_aux=False)
        outs = []
        for _ in range(2):
            dens = torch.full(dists.shape, float("nan"), device=G.DEV)
            col = torch.full(dists.shape + (3,), float("nan"), device=G.DEV)
            net.forward_rays_segment(*args, edge0, seg_len, None, None, dens, col)
            outs.append((dens, col))
    torch.cuda.synchronize()
    net.check_engine_status()
    seg = slice(edge0, edge0 + seg_len)
    (dens, col), (dens2, col2) = outs
    assert torch.equal(dens[:, seg], full["density"][:, seg])
    assert torch.equal(col[:, seg], full["color"][:, seg])
    assert torch.equal(dens[:, seg], dens2[:, seg]) and torch.equal(col[:, seg], col2[:, seg])
    for t in (dens, col):
        assert torch.isnan(t[:, :edge0]).all() and torch.isnan(t[:, edge0 + seg_len:]).all()
