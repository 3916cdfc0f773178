"""GPU: the NeRF tensor-core engine (csrc/nerf_tc.cu behind neddf_nerf_tc_*, engines "tc" and "auto" of
neddf_b200.NeRF) against the real-reference goldens, the fp64 oracle at every structure of tests/nerf_neus_configs.py and
the fp32 kernel; ragged sample counts, tile-mate independence, early ray termination, the fp16 range fallback and the
training path, which stays on the fp32 kernel."""
import json
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import neddf_oracle as orc  # noqa: E402
from tests import nerf_neus_configs as ncfg  # noqa: E402
from tests.field_configs import rays, samples  # noqa: E402
from tests.helpers import PARITY_TOL, nerr  # noqa: E402
from tests.test_nerf_gpu import build  # noqa: E402
from tests.test_nerf_oracle import NerfCase  # noqa: E402

DEV = torch.device("cuda:0")
GEOMETRY = (("point", 0.0), ("cone", orc.CONE_RAY_RADIUS))


def _report(**kw):
    print("NERF_TC " + json.dumps(kw))


def _net(name, engine="tc"):
    import neddf_b200
    net = neddf_b200.NeRF(**ncfg.kwargs(name))
    net.load_state_dict(ncfg.state_dict(name))
    net.to(DEV)
    net.set_iter(ncfg.CONFIGS[name]["iter"])
    net.engine = engine
    return net


def _golden(name, engine="tc"):
    render, cam = build(NerfCase(name))
    render.set_engine(engine)
    return render, cam


@pytest.mark.parametrize("name", ["relu", "tanhexp"])
def test_tc_field_and_render_rays_match_reference(name):
    import neddf_b200
    c = NerfCase(name)
    render, cam = _golden(name)
    assert render.network_fine.resolved_engine() == "tc"
    d, o = orc.make_rays(c.t("uv"), c.cam)
    radius = neddf_b200.ray.CONE_RAY_RADIUS if c.rc.sampling_type == "cone" else 0.0
    worst = 0.0
    for tag, net, dists in (("coarse", render.network_coarse, orc.coarse_dists(c.rc, c.t("u_coarse"))),
                            ("fine", render.network_fine, c.t("dists_fine"))):
        pos, dd, var = orc.make_samples(c.rc, d, o, dists)
        with torch.no_grad():
            out = net(neddf_b200.Sampling(pos.to(DEV), dd.contiguous().to(DEV), var.to(DEV)))
            fused = net.forward_rays(d.to(DEV), o.to(DEV), dists.to(DEV), c.rc.sampling_type, radius)
        for k in ("density", "color"):
            ref = c.z[f"field_{tag}_{k}"]
            for what, got in (("samples", out), ("fused", fused)):
                e = nerr(got[k].cpu().numpy(), ref)
                assert e < PARITY_TOL, (tag, k, what, e)
                worst = max(worst, e)
    with torch.no_grad():
        out = render.render_rays(c.t("uv").to(DEV), cam, uniforms=(c.t("u_coarse").to(DEV), c.t("u_fine").to(DEV)))
    for k in sorted(k[4:] for k in c.z if k.startswith("out_")):
        tol = 1e-3 if k.startswith("weight") else PARITY_TOL
        assert nerr(out[k].cpu().numpy(), c.z["out_" + k]) < tol, k
    render.check_status()
    _report(test="golden", name=name, worst_field=worst)


@pytest.mark.parametrize("name", ncfg.NERF)
def test_tc_structures_match_fp64_oracle_and_the_fp32_kernel(name):
    """forward and forward_rays (point and cone) at 1e-4 of the fp64 oracle; tc vs fp32 on the same samples within
    PARITY_TOL (the measured maximum is reported)."""
    import neddf_b200
    tc, fp = _net(name, "tc"), _net(name, "fp32")
    P = {k: v.double() for k, v in ncfg.params(name).items()}
    cfg, alpha = ncfg.config(name), ncfg.lowpass_alpha(name)
    seed = ncfg.SEED[name]
    pos, dd, var = samples(3, 700, seed)
    d, o, dists = rays(37, 29, seed + 1)
    worst, diff = 0.0, 0.0
    with torch.no_grad():
        cases = [("samples", (pos, dd, var), lambda n: n(neddf_b200.Sampling(pos.to(DEV), dd.to(DEV), var.to(DEV))))]
        for kind, radius in GEOMETRY:
            g = orc.point_samples(d, o, dists) if kind == "point" else orc.cone_samples(d, o, dists, radius)
            cases.append((kind, g, lambda n, kind=kind, radius=radius: n.forward_rays(d.to(DEV), o.to(DEV), dists.to(DEV),
                                                                                     kind, radius)))
        for what, (p3, d3, v3), run in cases:
            ref = orc.nerf_forward(P, cfg, alpha, p3.double(), d3.double(), v3.double())
            got, base = run(tc), run(fp)
            for k in ("density", "color"):
                e = nerr(got[k].cpu().numpy(), ref[k].numpy())
                assert e < PARITY_TOL, (name, what, k, e)
                worst = max(worst, e)
                de = nerr(got[k].cpu().numpy(), base[k].cpu().numpy())
                assert de < PARITY_TOL, (name, what, k, "tc vs fp32", de)
                diff = max(diff, de)
    tc.check_engine_status()
    _report(test="structures", name=name, worst_vs_fp64=worst, tc_vs_fp32=diff)


def test_tc_ragged_counts_leave_the_rest_untouched():
    """n in {0, 1, 127, 128, 129, 1000, 128 x 132 + 1} through the raw entry point into sentinel-filled outputs: the
    first n entries match the oracle, the rest keep the sentinel."""
    from neddf_b200 import _lib as L
    net = _net("N2_max_embed")
    P = {k: v.double() for k, v in ncfg.params("N2_max_embed").items()}
    cfg, alpha = ncfg.config("N2_max_embed"), ncfg.lowpass_alpha("N2_max_embed")
    N = 128 * 132 + 1
    pos, dd, var = samples(1, N + 7, 99)
    ref = orc.nerf_forward(P, cfg, alpha, pos.double(), dd.double(), var.double())
    pos_d, dd_d, var_d = (t.reshape(-1, 3).contiguous().to(DEV) for t in (pos, dd, var))
    h = net._field(DEV, kind=2)
    for n in (0, 1, 127, 128, 129, 1000, N):
        den = torch.full((N + 7,), 1234.5, device=DEV)
        col = torch.full((N + 7, 3), -777.0, device=DEV)
        L.check(L.lib().neddf_nerf_tc_forward(h, net._lowpass(), L.ptr(pos_d), L.ptr(dd_d), L.ptr(var_d), n, L.ptr(den),
                                              L.ptr(col), L.stream_ptr(DEV)), "nerf_tc_forward")
        torch.cuda.synchronize()
        if n:
            assert nerr(den[:n].cpu().numpy(), ref["density"].reshape(-1)[:n].numpy()) < PARITY_TOL, n
            assert nerr(col[:n].cpu().numpy(), ref["color"].reshape(-1, 3)[:n].numpy()) < PARITY_TOL, n
        assert bool((den[n:] == 1234.5).all()) and bool((col[n:] == -777.0).all()), n
    net.check_engine_status()


def test_tc_outputs_do_not_depend_on_tile_mates_or_the_call():
    """Chunked voxelize (1000-point launches) equals one launch over the grid bit for bit, a sample's outputs do not
    change when it moves within its tile, and two identical calls give identical outputs."""
    import neddf_b200
    net = _net("N4_deep_train")
    a = net.voxelize("density", cube_range=1.1, cube_resolution=41, chunk=1000)
    b = net.voxelize("density", cube_range=1.1, cube_resolution=41, chunk=41 ** 3)
    assert np.array_equal(a, b)
    pos, dd, var = (t.to(DEV) for t in samples(5, 999, 3))
    with torch.no_grad():
        x = net(neddf_b200.Sampling(pos, dd, var))
        y = net(neddf_b200.Sampling(pos, dd, var))
        # the same samples at other places in their tiles: shifted by 5
        s = net(neddf_b200.Sampling(pos.reshape(-1, 3)[5:].reshape(1, -1, 3), dd.reshape(-1, 3)[5:].reshape(1, -1, 3),
                                    var.reshape(-1, 3)[5:].reshape(1, -1, 3)))
    for k in ("density", "color"):
        assert torch.equal(x[k], y[k]), k
        assert torch.equal(x[k].reshape(5 * 999, -1)[5:], s[k].reshape(5 * 999 - 5, -1)), k
    net.check_engine_status()


def test_tc_segments_equal_the_whole_row_launch():
    """Every evaluated entry of forward_rays_segment equals forward_rays on engine "tc" bit for bit, over all rays and
    over a ray_index list with a device n_active, at several segments; entries outside stay untouched."""
    net = _net("N1_min")
    net2 = _net("N6_warmup")
    for n in (net, net2):
        d, o, dists = (t.to(DEV) for t in rays(300, 37, 5))
        B, E = dists.shape
        with torch.no_grad():
            full = n.forward_rays(d, o, dists, "cone", orc.CONE_RAY_RADIUS)
        idx = torch.tensor([299, 3, 0, 150, 7, 8, 200], dtype=torch.int32, device=DEV)
        for e0, seg in ((0, 1), (0, 37), (5, 11), (36, 1), (20, 17)):
            for ray_index, n_active in ((None, None), (idx, torch.tensor([5], dtype=torch.int32, device=DEV))):
                den = torch.full((B, E), -5.0, device=DEV)
                col = torch.full((B, E, 3), -5.0, device=DEV)
                with torch.no_grad():
                    n.forward_rays_segment(d, o, dists, "cone", orc.CONE_RAY_RADIUS, e0, seg, ray_index, n_active, den, col)
                rows = torch.arange(B, device=DEV) if ray_index is None else idx[:5].long()
                mask = torch.zeros(B, E, dtype=torch.bool, device=DEV)
                mask[rows.unsqueeze(1), torch.arange(e0, e0 + seg, device=DEV).unsqueeze(0)] = True
                assert torch.equal(den[mask], full["density"][mask]), (e0, seg)
                assert torch.equal(col[mask], full["color"][mask]), (e0, seg)
                assert bool((den[~mask] == -5.0).all()) and bool((col[~mask] == -5.0).all()), (e0, seg)
        n.check_engine_status()


@pytest.mark.parametrize("name", ["relu", "tanhexp"])
def test_tc_terminated_render_meets_count_and_bound(name, monkeypatch):
    """test_variant_termination_gpu's executed-count prediction and error bound on engine "tc"."""
    from tests import test_variant_termination_gpu as vt
    monkeypatch.setattr(vt, "_golden", lambda variant, n, sampling=None: _golden(n, "tc"))
    vt.test_executed_count_and_error_bound_when_rays_stop("nerf", name)


def _hot(engine):
    """The relu golden with outL_color.0's weight x 1e5 and 1e5 added to its bias: every sample's colour features leave
    fp16 range (densities stay sane), while the fp32 kernel still computes a finite colour."""
    render, cam = _golden("relu", engine)
    with torch.no_grad():
        for net in (render.network_coarse, render.network_fine):
            net.outL_color[0].weight.mul_(1e5)
            net.outL_color[0].bias.add_(1e5)
    return render, cam


def _image_uniforms(render, n_pix=40 * 30):
    g = torch.Generator().manual_seed(4)
    return (torch.rand(n_pix, render.sample_coarse + 1, generator=g).to(DEV),
            torch.rand(n_pix, render.sample_fine + 1, generator=g).to(DEV))


def test_tc_fp16_range_fallback():
    """"tc" raises FloatingPointError naming 65504; "auto" warns once, re-runs on fp32 with outputs equal to the fp32
    engine's in render_rays and render_image, and stays on fp32 afterwards."""
    c = NerfCase("relu")
    uv, u = c.t("uv").to(DEV), (c.t("u_coarse").to(DEV), c.t("u_fine").to(DEV))
    render, cam = _hot("tc")
    with torch.no_grad(), pytest.raises(FloatingPointError) as ei:
        render.render_rays(uv, cam, uniforms=u)
    assert "65504" in str(ei.value)
    ref_r, cam_r = _hot("fp32")
    with torch.no_grad():
        want = ref_r.render_rays(uv, cam_r, uniforms=u)
    want_img = ref_r.render_image(160, 120, cam_r, ["color", "depth"], 4, uniforms=_image_uniforms(ref_r))
    assert bool(torch.isfinite(want["color"]).all())
    for call in ("rays", "image"):
        render, cam = _hot("auto")
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            with torch.no_grad():
                got = (render.render_rays(uv, cam, uniforms=u) if call == "rays"
                       else render.render_image(160, 120, cam, ["color", "depth"], 4, uniforms=_image_uniforms(render)))
        assert sum(issubclass(x.category, RuntimeWarning) and "65504" in str(x.message) for x in w) == 1, call
        ref = want if call == "rays" else want_img
        for k in ref:
            assert torch.equal(got[k], ref[k]), (call, k)
        assert render.network_fine.resolved_engine() == "fp32" and render.network_coarse.resolved_engine() == "fp32"
        with warnings.catch_warnings():
            warnings.simplefilter("error")
            with torch.no_grad():
                again = render.render_rays(uv, cam, uniforms=u)
        for k in want:
            assert torch.equal(again[k], want[k]), k


def test_training_under_tc_equals_fp32():
    """training_kernels = True under "tc": loss and every gradient torch.equal to the same step under "fp32"."""
    c = NerfCase("relu")
    uv, u = c.t("uv").to(DEV), (c.t("u_coarse").to(DEV), c.t("u_fine").to(DEV))
    res = []
    for engine in ("fp32", "tc"):
        render, cam = _golden("relu", engine)
        for net in (render.network_coarse, render.network_fine):
            net.training_kernels = True
        out = render.render_rays(uv, cam, uniforms=u)
        loss = out["color"].square().mean() + out["depth"].mean() + out["color_coarse"].abs().mean()
        loss.backward()
        res.append((loss.detach(), [p.grad.clone() for p in render.parameters()]))
    assert torch.equal(res[0][0], res[1][0])
    assert len(res[0][1]) == len(res[1][1])
    for a, b in zip(res[0][1], res[1][1]):
        assert torch.equal(a, b)
