"""GPU parity tests: every kernel through the C ABI / host classes against the CPU oracle and the
golden vectors of the real reference.  Tolerance: 1e-4 tensor-normalised (BASELINE.json
north_star); searchsorted indices bit-exact given the same cdf."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import neddf_oracle as orc  # noqa: E402
from tests.helpers import PARITY_TOL, Case, assert_parity, nerr  # noqa: E402

CASES = ["bunny", "default", "point", "leaky"]
ENGINES = ["fp32", "tc", "tc2"]
GRAD_TOL = 1e-4  # north_star: 1e-4 rel fp32, gradients included


def _gpu():
    import tests.gpu_util as G
    return G


@pytest.mark.parametrize("n,k", [(128, 16), (128, 64), (128, 128), (16, 16), (16, 256)])
def test_tc_selftest_gemm(n, k):
    """wgmma building block (descriptor layouts, fp16-split 3-product accumulation) against an
    fp64 GEMM: hidden configuration (n=128) and head configuration (n=16)."""
    G = _gpu()
    from neddf_b200 import _lib as L
    g = torch.Generator().manual_seed(n * 1000 + k)
    a = torch.randn(128, k, generator=g)
    b = torch.randn(n, k, generator=g)
    a[3, 5 % k] = 300.0  # exercise a large magnitude (fp16 hi + lo)
    ad, bd = a.to(G.DEV), b.to(G.DEV)
    c = torch.full((128, n), float("nan"), device=G.DEV)
    L.check(L.lib().neddf_tc_selftest(L.ptr(ad), L.ptr(bd), 128, n, k, L.ptr(c), L.stream_ptr(G.DEV)), "tc_selftest")
    torch.cuda.synchronize()
    ref = a.double() @ b.double().T
    err = float((c.cpu().double() - ref).abs().max() / ref.abs().max())
    assert err < 2e-6, err


def test_make_rays_and_samples():
    G = _gpu()
    import neddf_b200
    c = Case("bunny")
    render, cam = G.build_render(c), G.build_camera(c)
    for dt in (torch.int64, torch.int32, torch.int16, torch.float32):
        rays = render.create_rays(c.t("uv").to(dt).to(G.DEV), cam)
        d_ref, o_ref = orc.make_rays(c.t("uv"), c.cam)
        assert nerr(rays.ray_dir.cpu().numpy(), d_ref.numpy()) < 1e-6
        assert nerr(rays.ray_orig.cpu().numpy(), o_ref.numpy()) == 0.0
    dists = orc.coarse_dists(c.rc, c.t("u_coarse"))
    for kind in ("cone", "point"):
        s = rays.get_sampling_cones(dists.to(G.DEV), neddf_b200.CONE_RAY_RADIUS) if kind == "cone" \
            else rays.get_sampling_points(dists.to(G.DEV))
        rc = orc.RenderConfig(sampling_type=kind)
        pos, d, var = orc.make_samples(rc, d_ref, o_ref, dists)
        assert nerr(s.sample_pos.cpu().numpy(), pos.numpy()) < 1e-6
        assert nerr(s.sample_dir.cpu().numpy(), d.numpy()) < 1e-6
        if kind == "cone":
            assert nerr(s.diag_variance.cpu().numpy(), var.numpy()) < 1e-5
        else:
            assert float(s.diag_variance.abs().max()) == 0.0


def test_coarse_dists_exact():
    G = _gpu()
    from neddf_b200 import _lib as L
    for (near, far, S) in ((2.0, 6.0, 64), (1.5, 5.5, 32), (0.1, 9.7, 100)):
        u = torch.rand(37, S + 1, generator=torch.Generator().manual_seed(5))
        ref = orc.coarse_dists(orc.RenderConfig(sample_coarse=S, dist_near=near, dist_far=far), u)
        ud = u.to(G.DEV)
        out = torch.empty_like(ud)
        L.check(L.lib().neddf_coarse_dists(L.ptr(ud), 37, S + 1, near, far, L.ptr(out), L.stream_ptr(G.DEV)))
        # same formula as torch.linspace + fp32 multiply-add; FMA contraction may move one ulp
        assert nerr(out.cpu().numpy(), ref.numpy()) < 2e-7


@pytest.mark.parametrize("name", CASES)
def test_composite_matches_reference(name):
    G = _gpu()
    c = Case(name)
    render = G.build_render(c)
    d_ref, o_ref = orc.make_rays(c.t("uv"), c.cam)
    for tag, dists in (("coarse", orc.coarse_dists(c.rc, c.t("u_coarse"))), ("fine", c.t("dists_fine"))):
        dens, col, pen = c.t(f"field_{tag}_density"), c.t(f"field_{tag}_color"), c.t(f"field_{tag}_fields_penalty")
        got = render.integrate_volume_render(dists.to(G.DEV), dens.to(G.DEV), col.to(G.DEV), pen.to(G.DEV))
        ref = orc.composite(dists, dens, col, c.rc.max_dist)
        ref["fields_penalty"] = orc.integrate_penalty(dists, pen)
        for k, v in ref.items():
            assert nerr(got[k].cpu().numpy(), v.numpy()) < 5e-6, (tag, k)
        if tag == "fine":  # and against the real reference's composited outputs
            for k in ("weight", "depth", "color", "transmittance", "fields_penalty"):
                assert nerr(got[k].cpu().numpy(), c.z["out_" + k]) < 1e-5, k
    render.check_status()


@pytest.mark.parametrize("name", CASES)
def test_sample_pdf_indices_bit_exact(name):
    G = _gpu()
    from neddf_b200 import _lib as L
    c = Case(name)
    render = G.build_render(c)
    dists = orc.coarse_dists(c.rc, c.t("u_coarse"))
    w = torch.from_numpy(c.z["out_weight_coarse"]).clone()
    u = c.t("u_fine")
    cdf = orc.pdf_cdf(w)
    new_ref, ids_ref = orc.invert_cdf(dists, cdf, u)
    B, E = dists.shape
    F = u.shape[1]
    ids = torch.empty(B, F, dtype=torch.int64, device=G.DEV)
    smp = torch.empty(B, F, dtype=torch.float32, device=G.DEV)
    dd, cd, ud = dists.to(G.DEV), cdf.to(G.DEV), u.to(G.DEV)  # keep alive across the raw-pointer call
    L.check(L.lib().neddf_invert_cdf(L.ptr(dd), L.ptr(cd), L.ptr(ud), B, E, F,
                                     L.ptr(smp), L.ptr(ids), L.stream_ptr(G.DEV)))
    assert torch.equal(ids.cpu(), ids_ref)  # bit-exact sample indices given the same cdf
    assert nerr(smp.cpu().numpy(), new_ref.numpy()) < 1e-6
    # full kernel: own cdf (fp64 scan), merge + sort
    wd = w.to(G.DEV).contiguous()
    out, ids2 = render.sample_pdf(dists.to(G.DEV), wd, F, uniform_rands=u.to(G.DEV), return_ids=True)
    ref = orc.sample_pdf(dists, w, u)
    # own cdf: torch's fp32 L1-norm reduction order is not reproducible (it differs from the
    # exactly rounded sum by a few ulp), which moves samples by <= ~5e-6 of the far distance
    assert nerr(out.cpu().numpy(), ref.numpy()) < 5e-6
    assert nerr(out.cpu().numpy(), c.z["dists_fine"]) < 5e-6
    mism = float((ids2.cpu() != ids_ref).float().mean())
    assert mism < 1e-3, mism  # cdf bits may differ in the last ulp from torch's summation order
    o = out.cpu()
    assert bool((o[:, 1:] >= o[:, :-1]).all())


def test_sample_pdf_sanitises_and_nan_fallback():
    G = _gpu()
    c = Case("bunny")
    render = G.build_render(c)
    dists = orc.coarse_dists(c.rc, c.t("u_coarse"))[:4]
    w = torch.rand(4, 64, generator=torch.Generator().manual_seed(1)) - 0.3
    w[1, 5] = float("nan")
    u = c.t("u_fine")[:4]
    wd = w.clone().to(G.DEV)
    out = render.sample_pdf(dists.to(G.DEV), wd, u.shape[1], uniform_rands=u.to(G.DEV))
    ref = orc.sample_pdf(dists, w.clone(), u)
    assert nerr(out.cpu().numpy(), ref.numpy()) < 5e-6
    assert torch.equal(wd.cpu(), orc.sanitise_weights(w))  # in-place side effect, base_neural_render.py:52-55
    # NaN distances -> batch-wide linspace fallback (base_neural_render.py:105-114)
    dn = dists.clone()
    dn[2, 10] = float("nan")
    out = render.sample_pdf(dn.to(G.DEV), w.clone().to(G.DEV), u.shape[1], uniform_rands=u.to(G.DEV))
    ref = torch.linspace(float(dn[0, 0]), float(dn[0, -1]), out.shape[1]).reshape(1, -1).expand(4, -1)
    assert nerr(out.cpu().numpy(), ref.numpy()) < 1e-6
    # the fallback is per launch like the reference's: a clean batch right after a NaN batch is resampled
    # normally although the host has not read/cleared the persistent flag yet
    assert int(render._status_buf[0].item()) & 2
    out = render.sample_pdf(dists.to(G.DEV), w.clone().to(G.DEV), u.shape[1], uniform_rands=u.to(G.DEV))
    assert nerr(out.cpu().numpy(), orc.sample_pdf(dists, w.clone(), u).numpy()) < 5e-6
    assert int(render._status_buf[0].item()) & 2  # still reported until check_status clears it
    render._status_buf.zero_()


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", CASES)
def test_field_forward_matches_reference(name, engine):
    """NeDDF.forward on the reference's own fine samples (Sampling tensors) vs the reference."""
    G = _gpu()
    import neddf_b200
    c = Case(name)
    render = G.build_render(c, engine)
    d_ref, o_ref = orc.make_rays(c.t("uv"), c.cam)
    pos, dd, var = orc.make_samples(c.rc, d_ref, o_ref, c.t("dists_fine"))
    with torch.no_grad():
        out = render.network_fine(neddf_b200.Sampling(pos.to(G.DEV), dd.contiguous().to(G.DEV), var.to(G.DEV)))
    for k in ("distance", "density", "color", "fields_penalty", "aux_grad"):
        assert_parity(out[k].cpu().numpy(), c.z["field_fine_" + k], PARITY_TOL, c.kinked, k)
    # ... and composited on the same fine distances it reproduces the reference's render outputs,
    # per-sample weights included
    comp = render.integrate_volume_render(c.t("dists_fine").to(G.DEV), out["density"], out["color"], out["fields_penalty"])
    for k in ("weight", "depth", "color", "transmittance", "fields_penalty"):
        assert_parity(comp[k].cpu().numpy(), c.z["out_" + k], PARITY_TOL, c.kinked, k)
    # fused-geometry entry point gives the same numbers
    with torch.no_grad():
        out2 = render.network_fine.forward_rays(d_ref.to(G.DEV), o_ref.to(G.DEV).contiguous(), c.t("dists_fine").to(G.DEV),
                                                c.rc.sampling_type, render._ray_radius, True, True)
    for k in ("distance", "density", "color", "fields_penalty", "aux_grad"):
        assert_parity(out2[k].cpu().numpy(), c.z["field_fine_" + k], PARITY_TOL, c.kinked, k)


@pytest.mark.parametrize("engine", ENGINES)
def test_field_forward_ragged_and_empty(engine):
    G = _gpu()
    import neddf_b200
    c = Case("default")
    render = G.build_render(c, engine)
    g = torch.Generator().manual_seed(3)
    for n in (0, 1, 15, 17, 16 * 148 + 5):
        pos = (torch.rand(1, n, 3, generator=g) - 0.5) * 2.0
        dd = torch.nn.functional.normalize(torch.randn(1, n, 3, generator=g), dim=-1)
        var = torch.rand(1, n, 3, generator=g) * 1e-3
        with torch.no_grad():
            out = render.network_fine(neddf_b200.Sampling(pos.to(G.DEV), dd.to(G.DEV), var.to(G.DEV)))
        assert out["density"].shape == (1, n)
        if n == 0:
            continue
        ref = orc.field_forward(c.p_fine, c.fc, c.st, pos, dd, var)
        for k, v in ref.items():
            assert nerr(out[k].cpu().numpy(), v.numpy()) < PARITY_TOL, (n, k)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", CASES)
def test_render_rays_matches_reference(name, engine):
    G = _gpu()
    c = Case(name)
    render, cam = G.build_render(c, engine), G.build_camera(c)
    with torch.no_grad():
        out = render.render_rays(c.t("uv").to(G.DEV), cam, uniforms=(c.t("u_coarse").to(G.DEV), c.t("u_fine").to(G.DEV)))
    ref = c.outputs()
    assert set(out.keys()) == set(ref.keys())
    for k, v in ref.items():
        assert tuple(out[k].shape) == v.shape, k
        # End to end, the per-sample fine `weight` is compared at positions that were themselves
        # resampled from the coarse weights: a 1e-6 change of a coarse weight moves fine samples,
        # and where two samples nearly coincide the interval width (hence the weight) moves by
        # far more in relative terms.  The integrated outputs keep the 1e-4 bound; the per-sample
        # weights are pinned at 1e-4 stage-wise (test_field_forward_matches_reference).
        tol = 1e-3 if k == "weight" else PARITY_TOL
        assert_parity(out[k].cpu().numpy(), v, tol, c.kinked, k)
    render.network_fine.check_engine_status()


@pytest.mark.parametrize("engine", ENGINES)
def test_render_image_matches_reference_image(engine):
    """bunny_smoke test frame 0 at downsampling 10 with the recorded uniforms: PSNR(new, ref)
    and PSNR vs ground truth like base_trainer.py:146-174."""
    import os
    G = _gpu()
    from tests.helpers import GOLDEN
    z = np.load(os.path.join(GOLDEN, "case_image.npz"))
    c = Case("bunny")
    render, cam = G.build_render(c, engine), G.build_camera(c)
    w, h, ds = int(z["width"]), int(z["height"]), int(z["downsampling"])
    n_pix = (w // ds) * (h // ds)
    g = torch.Generator().manual_seed(int(z["rand_seed"]))
    u_c = torch.rand(n_pix, 65, generator=g)
    u_f = torch.rand(n_pix, 129, generator=g)
    img = render.render_image(w, h, cam, ["color", "depth", "transmittance"], ds, 500, uniforms=(u_c, u_f))
    assert img["color"].shape == (h // ds, w // ds, 3) and img["depth"].shape == (h // ds, w // ds, 1)
    for k in ("color", "depth", "transmittance"):
        assert nerr(img[k].cpu().numpy(), z[k]) < PARITY_TOL, k
    mse = float(((img["color"].cpu().numpy().astype(np.float64) - z["color"]) ** 2).mean())
    psnr_new_ref = 10 * np.log10(1.0 / max(mse, 1e-30))
    assert psnr_new_ref > 80.0, psnr_new_ref
    rgb = np.clip(img["color"].cpu().numpy() * 255, 0, 255).astype(np.uint8)
    mse_gt = np.mean((rgb.astype(np.float64) - z["gt_bgr_u8"].astype(np.float64)) ** 2)
    assert 10 * np.log10(255.0 ** 2 / mse_gt) > 42.5  # reference: 43.09 dB
    assert render.network_fine.training and render.network_coarse.training  # nerf_render.py:247-248


def test_device_rng_default_and_determinism():
    G = _gpu()
    c = Case("bunny")
    render, cam = G.build_render(c), G.build_camera(c)
    uv = c.t("uv").to(G.DEV)
    with torch.no_grad():
        torch.manual_seed(0)
        a = render.render_rays(uv, cam)
        torch.manual_seed(0)
        b = render.render_rays(uv, cam)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert bool(torch.isfinite(a["color"]).all())


def test_errors_are_loud():
    G = _gpu()
    import neddf_b200
    c = Case("bunny")
    render, cam = G.build_render(c), G.build_camera(c)
    with pytest.raises(RuntimeError):
        render.render_rays(c.t("uv"), cam)  # CPU uv
    with pytest.raises(ValueError):
        with torch.no_grad():
            render.render_rays(c.t("uv").to(G.DEV), cam, uniforms=(torch.rand(3, 65), torch.rand(3, 129)))
    with pytest.raises(NotImplementedError):
        neddf_b200.NeRFRender(network_config={"_target_": "neddf.network.SomethingElse"})  # NeDDF, NeRF, NeuS are served


def _bench_render(engine):
    import bench
    import neddf_b200
    import tests.gpu_util as G
    sd, p = bench.seeded_state_dict()
    render = neddf_b200.NeRFRender(network_config=bench.NET_CFG, **bench.RENDER_CFG)
    render.load_state_dict(sd)
    render.to(G.DEV)
    render.set_iter(-1)
    render.set_engine(engine)
    R, T, calib = bench.synthetic_pose(0)
    cam = neddf_b200.Camera.from_matrix(neddf_b200.PinholeCalib(calib), R, T).to(G.DEV)
    cam.update_transform()
    return render, cam


def test_full_frame_properties():
    """BASELINE.json full size (800x800, 64+128): size-independent properties of the render."""
    import bench
    render, cam = _bench_render("auto")
    torch.manual_seed(0)
    img = render.render_image(bench.W, bench.H, cam, ["color", "depth", "transmittance"], 1, 1024)
    for k, c in (("color", 3), ("depth", 1), ("transmittance", 1)):
        assert img[k].shape == (bench.H, bench.W, c)
        assert bool(torch.isfinite(img[k]).all()), k
    t = img["transmittance"]
    assert float(t.min()) >= 0.0 and float(t.max()) <= 1.0 + 1e-3  # ReLU density: o in [0,1)
    d = img["depth"]
    assert float(d.min()) >= 2.0 - 1e-3 and float(d.max()) <= 6.1  # between near and max_dist


def test_partition_of_unity_and_sorted_samples_at_full_chunk():
    """sum(weights) + transmittance == 1 (up to the reference's +1e-7 per factor) on a 65,536-ray
    chunk; fine distances sorted and inside [near, far + jitter]."""
    import bench
    G = _gpu()
    render, cam = _bench_render("auto")
    n = 65536
    uv = orc.image_uv(bench.W, bench.H)[200 * bench.W:200 * bench.W + n].to(G.DEV)
    torch.manual_seed(1)
    with torch.no_grad():
        out = render.render_rays(uv, cam)
    s = out["weight"].sum(1) + out["transmittance"]
    assert float((s - 1).abs().max()) < 2e-4
    sc = out["weight_coarse"].sum(1) + out["transmittance_coarse"]
    assert float((sc - 1).abs().max()) < 1e-4
    assert bool((out["weight"] >= 0).all())


def test_engines_agree_on_bench_workload():
    """Tensor-core engines vs the fp32 FMA engine (device oracle) on 2,048 rays of the bench frame."""
    import bench
    G = _gpu()
    r_32, cam = _bench_render("fp32")
    n = 2048 + 37  # not a multiple of the 32- / 64-sample tiles
    uv = orc.image_uv(bench.W, bench.H)[400 * bench.W + 300:400 * bench.W + 300 + n].to(G.DEV)
    g = torch.Generator().manual_seed(2)
    u = (torch.rand(n, 65, generator=g).to(G.DEV), torch.rand(n, 129, generator=g).to(G.DEV))
    with torch.no_grad():
        b = r_32.render_rays(uv, cam, uniforms=u)
    for engine in ("tc", "tc2"):
        r_tc, _ = _bench_render(engine)
        with torch.no_grad():
            a = r_tc.render_rays(uv, cam, uniforms=u)
            a2 = r_tc.render_rays(uv, cam, uniforms=u)
        for k in ("color", "depth", "transmittance", "fields_penalty", "color_coarse", "weight_coarse"):
            assert nerr(a[k].cpu().numpy(), b[k].cpu().numpy()) < PARITY_TOL, (engine, k)
        for k in a:
            assert torch.equal(a[k], a2[k]), (engine, k)  # deterministic / idempotent


def test_point_sampling_against_oracle():
    """sampling_type="point" (the reference itself cannot run NeDDF in this mode - it calls .view on
    an expanded tensor, neddf.py:201 - so this branch is checked against the oracle only)."""
    G = _gpu()
    import neddf_b200
    c = Case("default")
    cfg = {k: v for k, v in dict(c.render_cfg, sampling_type="point").items() if k != "_target_"}
    rc = orc.RenderConfig(**cfg)
    render = neddf_b200.NeRFRender(network_config=c.net_cfg, **cfg)
    render.load_state_dict(c.state_dict())
    render.to(G.DEV)
    render.set_iter(-1)
    cam = G.build_camera(c)
    for engine in ENGINES:
        render.set_engine(engine)
        with torch.no_grad():
            out = render.render_rays(c.t("uv").to(G.DEV), cam, uniforms=(c.t("u_coarse").to(G.DEV), c.t("u_fine").to(G.DEV)))
        ref = orc.render_rays(c.p_coarse, c.p_fine, c.fc, c.st, rc, c.t("uv"), c.cam, c.t("u_coarse"), c.t("u_fine"))
        for k, v in ref.items():
            tol = 1e-3 if k == "weight" else PARITY_TOL
            assert nerr(out[k].cpu().numpy(), v.numpy()) < tol, (engine, k)


def test_voxelize_and_field_slice():
    """Secondary callers of NeDDF.forward (base_neuralfield.py:49-79, nerf_render.py:263-336)."""
    G = _gpu()
    c = Case("bunny")
    render = G.build_render(c, "auto")
    net = render.get_network()
    vox = net.voxelize("density", cube_range=1.1, cube_resolution=12, chunk=700)
    ids = np.linspace(-1.1, 1.1, 12)
    zs, ys, xs = np.meshgrid(ids, ids, ids)
    pos = torch.from_numpy(np.stack([xs.reshape(-1), ys.reshape(-1), zs.reshape(-1)], 1).astype(np.float32))[None]
    d = torch.tensor([1.0, 0.0, 0.0]).expand_as(pos)
    ref = orc.field_forward(c.p_fine, c.fc, c.st, pos, d, torch.zeros_like(pos))["density"].reshape(12, 12, 12)
    assert vox.shape == (12, 12, 12)
    assert nerr(vox, ref.numpy()) < PARITY_TOL
    fields = render.render_field_slice(0.0, 1.1, 32)
    assert set(fields) == {"distance", "density", "color", "aux_grad"}
    assert fields["distance"].shape == (32, 32, 3) and fields["distance"].dtype == np.uint8
    assert fields["color"].shape == (32, 32, 3)
    assert render.network_fine.training  # module mode untouched
    # values: the oracle on the same grid through the reference's scale table and colour map (nerf_render.py:295-334)
    import cv2
    lin = torch.linspace(-1.1, 1.1, 32)
    gx, gy = lin.reshape(1, -1).expand(32, 32), -lin.reshape(-1, 1).expand(32, 32)
    gpos = torch.stack([gx, gy, torch.zeros(32, 32)], 2).contiguous()
    gdir = torch.zeros_like(gpos)
    gdir[:, :, 2] = 1.0
    ref = orc.field_forward(c.p_fine, c.fc, c.st, gpos, gdir, torch.zeros_like(gpos))
    lut = cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(256, 1), cv2.COLORMAP_JET).reshape(256, 3).astype(np.int32)
    for key, scale in (("distance", 256.0), ("density", 12.8), ("color", 256.0), ("aux_grad", 256.0)):
        level = (scale * ref[key].reshape(32, 32, -1)).numpy().clip(0, 255).astype(np.uint8)
        got = fields[key]
        if level.shape[2] == 1:  # colour-mapped scalar field: recover the 8-bit level from the JET table
            got = np.abs(got.astype(np.int32)[:, :, None, :] - lut[None, None]).sum(-1).argmin(-1)[:, :, None]
        diff = np.abs(got.astype(np.int32) - level.astype(np.int32))
        assert diff.max() <= 1 and (diff == 0).mean() > 0.97, (key, int(diff.max()), float((diff == 0).mean()))


@pytest.mark.parametrize("engine", ENGINES)
def test_training_state_forward_values(engine):
    """Warm-up scalars of NeDDF.set_iter(3000) (aux_grad_scale 0.3, neddf.py:323-326): forward
    values against the reference's grad-mode run (golden case_train), forward only (the gradients of the same
    case are held to the reference's by test_render_rays_training_matches_reference_gradients)."""
    G = _gpu()
    c = Case("train")
    render, cam = G.build_render(c, engine), G.build_camera(c)
    assert render.iteration == 3000 and abs(render.network_fine.aux_grad_scale - 0.3) < 1e-12
    with torch.no_grad():
        out = render.render_rays(c.t("uv").to(G.DEV), cam, uniforms=(c.t("u_coarse").to(G.DEV), c.t("u_fine").to(G.DEV)))
    for k, v in c.outputs().items():
        tol = 1e-3 if k == "weight" else PARITY_TOL
        assert nerr(out[k].cpu().numpy(), v) < tol, k


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("n_rays", [1, 3, 33])
def test_render_rays_ragged_batches(engine, n_rays):
    """Batches that do not fill a 32-sample tile / 16-sample tile evenly."""
    G = _gpu()
    c = Case("default")
    render, cam = G.build_render(c, engine), G.build_camera(c)
    g = torch.Generator().manual_seed(n_rays)
    uv = torch.randint(200, 600, (n_rays, 2), generator=g)
    u_c, u_f = torch.rand(n_rays, 65, generator=g), torch.rand(n_rays, 129, generator=g)
    with torch.no_grad():
        out = render.render_rays(uv.to(G.DEV), cam, uniforms=(u_c.to(G.DEV), u_f.to(G.DEV)))
    ref = orc.render_rays(c.p_coarse, c.p_fine, c.fc, c.st, c.rc, uv, c.cam, u_c, u_f)
    for k, v in ref.items():
        tol = 1e-3 if k == "weight" else PARITY_TOL
        assert nerr(out[k].cpu().numpy(), v.numpy()) < tol, (n_rays, k)


def test_weights_repacked_after_in_place_update():
    """Optimisers update parameters in place: the packed kernel weights must follow
    (neddf_field_set_weights is re-run when a parameter's version counter changes)."""
    G = _gpu()
    import neddf_b200
    c = Case("default")
    render, cam = G.build_render(c, "auto"), G.build_camera(c)
    uv = c.t("uv").to(G.DEV)
    u = (c.t("u_coarse").to(G.DEV), c.t("u_fine").to(G.DEV))
    with torch.no_grad():
        a = render.render_rays(uv, cam, uniforms=u)
        for p in render.get_parameters_list():
            p.mul_(1.01)
        b = render.render_rays(uv, cam, uniforms=u)
    assert not torch.equal(a["color"], b["color"])
    p2 = {k: v * 1.01 for k, v in c.p_fine.items()}
    ref = orc.render_rays(p2, p2, c.fc, c.st, c.rc, c.t("uv"), c.cam, c.t("u_coarse"), c.t("u_fine"))
    for k in ("color", "depth", "transmittance"):
        assert nerr(b[k].cpu().numpy(), ref[k].numpy()) < PARITY_TOL, k


@pytest.mark.parametrize("name", ["bunny", "default"])
def test_composite_backward_matches_autograd(name):
    """neddf_composite_backward against autograd through the oracle's restatement of
    integrate_volume_render + penalty integration (what the reference's training step
    differentiates, base_neural_render.py:148-172, nerf_render.py:153-159)."""
    G = _gpu()
    c = Case(name)
    render = G.build_render(c)
    dists = c.t("dists_fine")
    dens = c.t("field_fine_density").clone().requires_grad_(True)
    col = c.t("field_fine_color").clone().requires_grad_(True)
    pen = c.t("field_fine_fields_penalty").clone().requires_grad_(True)
    g = torch.Generator().manual_seed(9)
    B, E = dists.shape
    gw, gd, gc = torch.randn(B, E - 1, generator=g), torch.randn(B, generator=g), torch.randn(B, 3, generator=g)
    gt, gp = torch.randn(B, generator=g), torch.randn(B, generator=g)
    ref = orc.composite(dists, dens, col, c.rc.max_dist)
    ref_pen = orc.integrate_penalty(dists, pen)
    loss = (ref["weight"] * gw).sum() + (ref["depth"] * gd).sum() + (ref["color"] * gc).sum() + \
        (ref["transmittance"] * gt).sum() + (ref_pen * gp).sum()
    loss.backward()
    dd = dens.detach().to(G.DEV).requires_grad_(True)
    cd = col.detach().to(G.DEV).requires_grad_(True)
    pd = pen.detach().to(G.DEV).requires_grad_(True)
    out = render.integrate_volume_render(dists.to(G.DEV), dd, cd, pd)
    l2 = (out["weight"] * gw.to(G.DEV)).sum() + (out["depth"] * gd.to(G.DEV)).sum() + (out["color"] * gc.to(G.DEV)).sum() + \
        (out["transmittance"] * gt.to(G.DEV)).sum() + (out["fields_penalty"] * gp.to(G.DEV)).sum()
    l2.backward()
    assert abs(float(l2) - float(loss)) < 1e-4 * abs(float(loss)) + 1e-5
    assert nerr(dd.grad.cpu().numpy(), dens.grad.numpy()) < 2e-5
    assert nerr(cd.grad.cpu().numpy(), col.grad.numpy()) < 2e-5
    assert nerr(pd.grad.cpu().numpy(), pen.grad.numpy()) < 2e-5
    assert float(dd.grad[:, -1].abs().max()) == 0.0  # the closing edge receives no gradient


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", ["train", "bunny"])
def test_field_backward_matches_autograd(name, engine):
    """Training path of the field (neddf_field_forward_train of the module's engine + neddf_field_backward +
    weight gradients) against autograd through the oracle, for random upstream gradients of density,
    colour and fields_penalty."""
    G = _gpu()
    c = Case(name)
    render = G.build_render(c, engine)
    net = render.network_fine
    n_rays = 6
    d, o = orc.make_rays(c.t("uv")[:n_rays], c.cam)
    dists = c.t("dists_fine")[:n_rays, ::3].contiguous()
    pos, dd, var = orc.make_samples(c.rc, d, o, dists)
    g = torch.Generator().manual_seed(4)
    B, S = dists.shape
    gd, gc, gp = torch.randn(B, S, generator=g), torch.randn(B, S, 3, generator=g), torch.randn(B, S, generator=g)
    Pg = {k: v.clone().requires_grad_(True) for k, v in c.p_fine.items()}
    ref = orc.field_forward(Pg, c.fc, c.st, pos, dd.contiguous(), var)
    ((ref["density"] * gd).sum() + (ref["color"] * gc).sum() + (ref["fields_penalty"] * gp).sum()).backward()
    out = net.forward_rays(d.contiguous().to(G.DEV), o.contiguous().to(G.DEV), dists.to(G.DEV), c.rc.sampling_type,
                           render._ray_radius)
    for k in ("density", "color", "fields_penalty"):
        assert nerr(out[k].detach().cpu().numpy(), ref[k].detach().numpy()) < PARITY_TOL, k
    loss = (out["density"] * gd.to(G.DEV)).sum() + (out["color"] * gc.to(G.DEV)).sum() + \
        (out["fields_penalty"] * gp.to(G.DEV)).sum()
    net.zero_grad()
    loss.backward()
    for k, v in Pg.items():
        mod, attr = k.rsplit(".", 1)
        obj = net
        for part in mod.split("."):
            obj = obj[int(part)] if part.isdigit() else getattr(obj, part)
        got = getattr(obj, attr).grad
        assert got is not None, k
        # measured (tools/grad_err.py): 1.6e-6 .. 3.5e-5 against the fp64 arbiter on all three engines; the
        # fp32 reference itself sits at 1e-6 .. 1e-5 of fp64 (tests/test_oracle_derivatives.py)
        assert nerr(got.cpu().numpy(), v.grad.numpy()) < GRAD_TOL, k


def test_render_rays_training_matches_reference_gradients():
    """drums-config inner loop (forward + backward) on the golden training case: outputs and the
    parameter gradients of the reference's own backward (hand-written autograd Functions,
    run.py / nerf_trainer.py:108-122) for the recorded loss."""
    G = _gpu()
    c = Case("train")
    render, cam = G.build_render(c, "auto"), G.build_camera(c)
    out = render.render_rays(c.t("uv").to(G.DEV), cam, uniforms=(c.t("u_coarse").to(G.DEV), c.t("u_fine").to(G.DEV)))
    for k, v in c.outputs().items():
        tol = 1e-3 if k == "weight" else PARITY_TOL
        assert nerr(out[k].detach().cpu().numpy(), v) < tol, k
    loss = (out["color"].sum() + 0.1 * out["depth"].sum() + 0.05 * out["transmittance"].sum()
            + 0.01 * out["fields_penalty"].sum() + 0.1 * out["color_coarse"].sum()
            + 0.001 * out["fields_penalty_coarse"].sum())
    assert abs(float(loss) - float(c.z["loss"])) < 1e-4 * abs(float(c.z["loss"]))
    render.zero_grad()
    loss.backward()
    checked = 0
    for name, p in render.named_parameters():
        key = "grad_" + name
        if key not in c.z:
            key = "grad_" + name.replace("network_fine.", "network_coarse.")
        ref = c.z[key]
        g = p.grad.cpu().numpy()
        if g.ndim == 2 and g.shape[1] > 3:
            g = g[::8]
        assert nerr(g, ref) < 2 * GRAD_TOL, name  # end to end: resampled positions move with the coarse weights
        checked += 1
    assert checked == 26


def test_network_forward_sampling_is_differentiable():
    """NeDDF.forward(Sampling) under autograd (the reference's trainer test runs exactly this through
    render_rays; direct callers get the same differentiable path): values and parameter gradients
    against autograd through the oracle."""
    G = _gpu()
    import neddf_b200
    c = Case("default")
    render = G.build_render(c, "auto")
    net = render.network_fine
    g = torch.Generator().manual_seed(11)
    B, S = 3, 21
    pos = (torch.rand(B, S, 3, generator=g) - 0.5) * 2.0
    dd = torch.nn.functional.normalize(torch.randn(B, S, 3, generator=g), dim=-1)
    var = torch.rand(B, S, 3, generator=g) * 1e-3
    gd, gc, gp = torch.randn(B, S, generator=g), torch.randn(B, S, 3, generator=g), torch.randn(B, S, generator=g)
    Pg = {k: v.clone().requires_grad_(True) for k, v in c.p_fine.items()}
    ref = orc.field_forward(Pg, c.fc, c.st, pos, dd, var)
    ((ref["density"] * gd).sum() + (ref["color"] * gc).sum() + (ref["fields_penalty"] * gp).sum()).backward()
    out = net(neddf_b200.Sampling(pos.to(G.DEV), dd.to(G.DEV), var.to(G.DEV)))
    assert set(out) == {"distance", "density", "color", "fields_penalty", "aux_grad"}
    for k in out:
        assert nerr(out[k].detach().cpu().numpy(), ref[k].detach().numpy()) < PARITY_TOL, k
    assert out["density"].requires_grad and not out["distance"].requires_grad
    net.zero_grad()
    ((out["density"] * gd.to(G.DEV)).sum() + (out["color"] * gc.to(G.DEV)).sum() + (out["fields_penalty"] * gp.to(G.DEV)).sum()).backward()
    for k in ("layers_ddf.0.weight", "layers_ddf.5.weight", "layers_col.0.weight", "layer_ddf_out.weight",
              "layer_aux_out.bias", "layer_col_out.weight", "layers_ddf.6.bias"):
        mod, attr = k.rsplit(".", 1)
        obj = net
        for part in mod.split("."):
            obj = obj[int(part)] if part.isdigit() else getattr(obj, part)
        assert nerr(getattr(obj, attr).grad.cpu().numpy(), Pg[k].grad.numpy()) < GRAD_TOL, k


def test_other_embedding_ranks_run_on_a_tensor_core_engine():
    """The reference's own test fixture uses embed_pos_rank=6 (tests/conftest.py:77-99); both tensor-core engines cover
    any ranks whose inputs fit AUX: "auto" must not fall to the slower fp32 engine, and the results of "auto" (the
    single-CTA engine) and of the CTA-pair engine must match the oracle."""
    G = _gpu()
    import neddf_b200
    cfg = dict(embed_pos_rank=6, embed_dir_rank=2, ddf_layer_count=5, col_layer_count=3, skips=[1],
               activation_type="tanhExp", density_activation_type="LeakyReLU", d_near=0.01, lowpass_alpha_offset=6.0)
    fc = orc.FieldConfig(**cfg)
    P = orc.init_params(fc, 5, bias_std=0.05)
    net = neddf_b200.NeDDF(**cfg)
    net.load_state_dict(P)
    net.to(G.DEV)
    net.set_iter(-1)
    assert net.resolved_engine() == "tc"
    g = torch.Generator().manual_seed(3)
    B, S = 5, 37
    pos = (torch.rand(B, S, 3, generator=g) - 0.5) * 2.0
    dd = torch.nn.functional.normalize(torch.randn(B, S, 3, generator=g), dim=-1)
    var = torch.rand(B, S, 3, generator=g) * 1e-3
    st = orc.FieldState.at_iter(fc, -1)
    with torch.no_grad():
        ref = orc.field_forward(P, fc, st, pos, dd, var)
    for engine in ("auto", "tc2"):
        net.engine = engine
        with torch.no_grad():
            out = net(neddf_b200.Sampling(pos.to(G.DEV), dd.to(G.DEV), var.to(G.DEV)))
        for k in ("distance", "density", "color", "fields_penalty", "aux_grad"):
            assert nerr(out[k].cpu().numpy(), ref[k].numpy()) < PARITY_TOL, (engine, k)
        net.check_engine_status()


@pytest.mark.parametrize("engine", ["tc", "tc2", "fp32"])
def test_early_ray_termination(engine):
    """Opt-in early ray termination of the fine pass (BASELINE.json configs[4]; the reference has none):
    off = the normal path; one segment = the segment kernel on all samples = bit-identical outputs; on =
    bounded error (|d color| <= eps max|c|, |d depth| <= eps max_dist, |d T| <= eps) and fewer evaluations."""
    G = _gpu()
    import os
    from tests.helpers import GOLDEN
    z = np.load(os.path.join(GOLDEN, "case_image.npz"))
    c = Case("bunny")
    render, cam = G.build_render(c, engine), G.build_camera(c)
    w, h, ds = int(z["width"]), int(z["height"]), int(z["downsampling"])
    n_pix = (w // ds) * (h // ds)
    g = torch.Generator().manual_seed(int(z["rand_seed"]))
    u = (torch.rand(n_pix, 65, generator=g).to(G.DEV), torch.rand(n_pix, 129, generator=g).to(G.DEV))
    keys = ["color", "depth", "transmittance"]
    base = render.render_image(w, h, cam, keys, ds, uniforms=u)
    assert render.termination_stats() == {"executed": 0, "nominal": 0}
    render.transmittance_eps, render.termination_segments = 1e-30, 1  # one segment: nothing can stop early
    one = render.render_image(w, h, cam, keys, ds, uniforms=u)
    st = render.termination_stats()
    assert st["executed"] == st["nominal"] > 0
    for k in keys:
        assert torch.equal(one[k], base[k]), k
    cmax = float(base["color"].abs().max())
    saved = []
    for eps in (1e-3, 5e-2):  # (the smoke bunny is translucent: few rays ever get below 1e-3)
        render.transmittance_eps, render.termination_segments = eps, 6
        out = render.render_image(w, h, cam, keys, ds, uniforms=u)
        st = render.termination_stats()
        assert 0 < st["executed"] <= st["nominal"], st
        saved.append(1.0 - st["executed"] / st["nominal"])
        assert float((out["color"] - base["color"]).abs().max()) <= eps * cmax * 1.05 + 1e-6
        assert float((out["depth"] - base["depth"]).abs().max()) <= eps * render.max_dist * 1.05 + 1e-6
        assert float((out["transmittance"] - base["transmittance"]).abs().max()) <= eps * 1.05
    assert saved[1] >= saved[0] > 0.0, saved
    render.check_status()


def test_terminate_rays_kernel():
    """neddf_terminate_rays on a synthetic wall: transmittance update = the compositing factors
    (base_neural_render.py:148-160), kept rays = exactly those with T > eps, executed-evaluation counter."""
    G = _gpu()
    from neddf_b200 import _lib as L
    g = torch.Generator().manual_seed(8)
    B, E = 1000, 40
    dists = torch.sort(torch.rand(B, E, generator=g) * 4 + 2, dim=1).values
    dens = torch.rand(B, E, generator=g) * 0.3
    dens[::3, 10:14] = 80.0  # an opaque wall on every third ray
    o = 1 - torch.exp(-dens[:, :-1] * (dists[:, 1:] - dists[:, :-1]))
    fac = 1 - o + 1e-7
    dd, sd = dists.to(G.DEV), dens.to(G.DEV)
    trans = torch.ones(B, device=G.DEV)
    idx = [torch.full((B,), -1, dtype=torch.int32, device=G.DEV) for _ in range(2)]
    cnt = [torch.zeros(1, dtype=torch.int32, device=G.DEV) for _ in range(2)]
    ex = torch.zeros(1, dtype=torch.int64, device=G.DEV)
    eps = 1e-2
    cur_i, cur_n, live, expect_ex = None, None, torch.ones(B, dtype=torch.bool), 0
    T = torch.ones(B)
    for k, (e0, seg) in enumerate(((0, 12), (12, 12), (24, 16))):
        L.check(L.lib().neddf_terminate_rays(L.ptr(dd), L.ptr(sd), B, E, e0, seg, L.ptr(cur_i), L.ptr(cur_n), L.ptr(trans), eps,
                                             L.ptr(idx[k % 2]), L.ptr(cnt[k % 2]), L.ptr(ex), L.stream_ptr(G.DEV)))
        torch.cuda.synchronize()
        expect_ex += int(live.sum()) * seg
        e1 = min(e0 + seg, E - 1)
        T = torch.where(live, T * fac[:, e0:e1].prod(1), T)
        live = live & (T > eps)
        n = int(cnt[k % 2].item())
        kept = torch.sort(idx[k % 2][:n].cpu().long()).values
        assert torch.equal(kept, torch.nonzero(live).flatten()), k
        assert nerr(trans.cpu().numpy(), T.numpy()) < 1e-5
        cur_i, cur_n = idx[k % 2], cnt[k % 2]
    assert int(ex.item()) == expect_ex
    assert int((~live).sum()) >= B // 3  # the walls stopped their rays


@pytest.mark.parametrize("rows,lda,col0,ka", [(4096, 256, 0, 128), (100003, 256, 128, 128), (7777, 60, 0, 60), (5000, 87, 0, 87),
                                              (9001, 2, 0, 2), (6000, 4, 0, 3)])
def test_wgrad_gemm(rows, lda, col0, ka):
    """neddf_wgrad (wgmma split-K GEMM, fp16 hi/lo operands split on the fly) against an fp64 matmul:
    the shapes of the training backward (aligned / ragged / 2- and 3-column head operands, slab remainders)."""
    G = _gpu()
    from neddf_b200 import _lib as L
    g = torch.Generator().manual_seed(rows + ka)
    A = torch.randn(rows, lda, generator=g)
    B = torch.randn(rows, 256, generator=g)
    A[5 % rows, col0] = 300.0
    Ad, Bd = A.to(G.DEV), B.to(G.DEV)
    out = torch.full((ka, 256), float("nan"), device=G.DEV)
    ws = torch.empty(int(L.lib().neddf_wgrad_workspace_bytes()) // 4, device=G.DEV)
    L.check(L.lib().neddf_wgrad(L.ptr(Ad), lda, col0, ka, L.ptr(Bd), 256, rows, L.ptr(out), 256, 256, L.ptr(ws),
                                L.stream_ptr(G.DEV)), "wgrad")
    out2 = torch.empty_like(out)
    L.check(L.lib().neddf_wgrad(L.ptr(Ad), lda, col0, ka, L.ptr(Bd), 256, rows, L.ptr(out2), 256, 256, L.ptr(ws),
                                L.stream_ptr(G.DEV)), "wgrad")
    torch.cuda.synchronize()
    ref = A[:, col0:col0 + ka].double().t() @ B.double()
    err = float((out.cpu().double() - ref).abs().max() / ref.abs().max())
    assert err < 1e-5, err  # fp32 accumulation over up to 1e5 rows (the split operands themselves are good to 2e-7)
    assert torch.equal(out, out2)  # fixed summation order
    gsum = torch.empty(256, device=G.DEV)
    n_s = rows // 4
    L.check(L.lib().neddf_colsum_value_rows(L.ptr(Bd), n_s, 4 * 256, L.ptr(gsum), L.ptr(ws), L.stream_ptr(G.DEV)), "colsum")
    refs = B[:4 * n_s].reshape(n_s, 4, 256)[:, 0, :].double().sum(0)
    assert float((gsum.cpu().double() - refs).abs().max() / refs.abs().max()) < 1e-5


def test_fused_losses_match_the_reference_objective():
    """neddf_render_loss (values + gradients of the reference's objective, loss/*.py) against plain torch ops."""
    G = _gpu()
    import bench
    from neddf_b200 import losses
    g = torch.Generator().manual_seed(21)
    B = 777
    mk = lambda *s: torch.rand(*s, generator=g).to(G.DEV).requires_grad_(True)  # noqa: E731
    out = {"color": mk(B, 3), "color_coarse": mk(B, 3), "transmittance": mk(B), "transmittance_coarse": mk(B),
           "fields_penalty": mk(B), "fields_penalty_coarse": mk(B)}
    with torch.no_grad():
        out["transmittance"][:5] = torch.tensor([0.0, 1.0, 1e-8, 1 - 1e-8, 0.5])  # both sides of the clamp
    tgt = {"color": torch.rand(B, 3, generator=g).to(G.DEV), "mask": (torch.rand(B, generator=g) > 0.4).float().to(G.DEV)}
    ref = bench.train_loss(out, tgt["color"], tgt["mask"])
    ref.backward()
    gref = {k: v.grad.clone() for k, v in out.items()}
    for v in out.values():
        v.grad = None
    d = losses.RenderLoss()(out, tgt)
    assert list(d) == ["color", "color_coarse", "mask", "mask_coarse", "fields_penalty", "fields_penalty_coarse"]
    total = torch.sum(torch.stack(list(d.values())))  # nerf_trainer.py:121
    assert abs(float(total) - float(ref)) < 1e-6 * abs(float(ref))
    total.backward()
    for k, v in out.items():
        assert nerr(v.grad.cpu().numpy(), gref[k].cpu().numpy()) < 1e-6, k
    # the three drop-in classes: same dictionary, one term pair each
    for v in out.values():
        v.grad = None
    parts = {}
    for cls, w in ((losses.ColorLoss, (1.0, 0.1)), (losses.MaskBCELoss, (0.05, 0.005)), (losses.FieldsConstraintLoss, (0.01, 0.01))):
        parts.update(cls(*w)(out, tgt))
    for k in d:
        assert abs(float(parts[k]) - float(d[k])) <= 1e-7 * abs(float(d[k])) + 1e-12, k
    assert "color_coarse" not in losses.ColorLoss(1.0, 0.0)(out, tgt)  # base_loss.py:76


def test_fused_adam_matches_torch_adam_and_repacks():
    """FusedAdam (one launch per network + re-pack on the same stream) against torch.optim.Adam over three
    training steps: parameters agree, and the next forward uses the updated (re-packed) weights."""
    G = _gpu()
    import bench
    import neddf_b200
    from neddf_b200 import losses, optim
    c = Case("train")
    cam = G.build_camera(c)
    uv = c.t("uv").to(G.DEV)
    u = (c.t("u_coarse").to(G.DEV), c.t("u_fine").to(G.DEV))
    tgt = {"color": torch.rand(uv.shape[0], 3, generator=torch.Generator().manual_seed(1)).to(G.DEV),
           "mask": torch.ones(uv.shape[0], device=G.DEV)}
    loss_fn = losses.RenderLoss()
    renders, opts = [], []
    for fused in (False, True):
        r = G.build_render(c, "auto")
        o = optim.FusedAdam.for_render(r, lr=5e-4) if fused else torch.optim.Adam(r.get_parameters_list(), lr=5e-4)
        renders.append(r)
        opts.append(o)
    # identical gradients go to both optimisers (Adam's normalised update amplifies 1e-7 gradient noise to
    # 1e-4 parameter differences within two steps, so re-deriving the gradients from each model's own weights
    # would test the conditioning of the scene, not the optimiser)
    for it in range(3):
        r0 = renders[0]
        r0.set_iter(c.iter + it)
        out = r0.render_rays(uv, cam, uniforms=u)
        loss = torch.sum(torch.stack(list(loss_fn(out, tgt).values())))
        opts[0].zero_grad(set_to_none=True)
        loss.backward()
        for p0, p1 in zip(renders[0].parameters(), renders[1].parameters()):
            p1.grad = p0.grad.clone()
        opts[0].step()
        opts[1].step()
        for (n0, p0), (n1, p1) in zip(renders[0].named_parameters(), renders[1].named_parameters()):
            assert n0 == n1
            assert nerr(p1.detach().cpu().numpy(), p0.detach().cpu().numpy()) < 1e-6, (it, n0)
    renders[1].set_iter(c.iter + 2)
    with torch.no_grad():
        a = renders[0].render_rays(uv, cam, uniforms=u)
        b = renders[1].render_rays(uv, cam, uniforms=u)
    for k in ("color", "depth", "fields_penalty"):
        assert nerr(b[k].cpu().numpy(), a[k].cpu().numpy()) < 1e-5, k


def test_sample_pdf_without_coarse_edges():
    """sample_pdf(cat_coarse=False) (base_neural_render.py:61-68, 104) against the real reference's golden
    output and the oracle; in-place sanitising of the weights as in the other mode."""
    G = _gpu()
    import os
    from tests.helpers import GOLDEN
    z = np.load(os.path.join(GOLDEN, "case_pdf_nocat.npz"))
    c = Case("bunny")
    render = G.build_render(c)
    wd = torch.from_numpy(z["weights"]).clone().to(G.DEV)
    out = render.sample_pdf(torch.from_numpy(z["dists"]).to(G.DEV), wd, z["u"].shape[1], cat_coarse=False,
                            uniform_rands=torch.from_numpy(z["u"]).to(G.DEV))
    assert out.shape == z["out"].shape
    assert nerr(out.cpu().numpy(), z["out"]) < 5e-6
    assert np.array_equal(wd.cpu().numpy(), z["weights_after"], equal_nan=True)
    o = out.cpu()
    assert bool((o[:, 1:] >= o[:, :-1]).all())
    render._status_buf.zero_()


@pytest.mark.parametrize("case,n_rays", [("bunny", 1), ("bunny", 3), ("bunny", 37), ("bunny", 600), ("bunny", 2500),
                                         ("default", 600), ("point", 600), ("leaky", 600)])
def test_tc_images_only_colour_trunk_matches_full_program(case, n_rays):
    """Images-only launches of the tc engine (no fields_penalty) run the colour trunk on the 32 value rows of a tile
    (N = 32 MMAs, DESIGN 4.1).  Same results as the full program (N = 128, Jacobian rows included) for launches with
    fewer tiles than CTAs, ragged last tiles and several tiles per CTA, for every golden configuration (activations,
    skips, sampling types), and as the oracle (neddf.py:200-257 through oracle.field_forward)."""
    import neddf_b200
    G = _gpu()
    c = Case(case)
    render = G.build_render(c, "tc")
    net = render.network_fine
    assert net.resolved_engine(G.DEV) == "tc"
    g = torch.Generator().manual_seed(n_rays)
    uv = torch.stack([torch.randint(0, 50, (n_rays,), generator=g), torch.randint(0, 50, (n_rays,), generator=g)], 1).float()
    d, o = orc.make_rays(uv, c.cam)
    dists = orc.coarse_dists(c.rc, torch.rand(n_rays, c.rc.sample_coarse + 1, generator=g))
    radius = neddf_b200.ray.CONE_RAY_RADIUS if c.rc.sampling_type == "cone" else 0.0

    def run(need_penalty):
        with torch.no_grad():
            out = net.forward_rays(d.to(G.DEV), o.to(G.DEV), dists.to(G.DEV), c.rc.sampling_type, radius,
                                   need_penalty=need_penalty, need_aux=True)
        torch.cuda.synchronize()
        net.check_engine_status()
        return {k: v.cpu() for k, v in out.items()}

    images = run(False)
    full = run(True)
    for k in ("density", "distance", "aux_grad"):
        assert torch.equal(images[k], full[k]), k  # the distance trunk is the same program
    # colour: N = 32 instead of N = 128 MMAs over the same value rows
    assert nerr(images["color"].numpy(), full["color"].numpy()) < 1e-6
    pos, dd, var = orc.make_samples(c.rc, d, o, dists)
    with torch.no_grad():
        ref = orc.field_forward(c.p_fine, c.fc, c.st, pos, dd, var)
    # (random pixels mostly look past the bunny: densities of 1e-2 and below, for which max|ref| is no scale -
    # the floor of 1 keeps the bound absolute there; colours are O(1))
    for k in ("density", "color"):
        a, r = images[k].numpy(), ref[k].numpy()
        e = np.abs(a.astype(np.float64) - r) / max(np.abs(r).max(), 1.0)
        if c.kinked:  # same allowance as helpers.assert_parity: the few samples within rounding distance of a kink
            assert int((e >= PARITY_TOL).sum()) <= max(2, int(1e-2 * e.size)) and e.max() < 5e-2, (k, e.max())
        else:
            assert e.max() < PARITY_TOL, (k, e.max())


def test_auto_engine_leaves_fp16_range_gracefully():
    """Engine cliff (VERDICT round 1, weak 9): weights that push a hidden activation beyond fp16 range (65504, the
    limit of the tensor-core engine's split operands).  Explicit "tc" / "tc2" raise; "auto" switches the network to
    the fp32 engine, warns and re-runs the call - same rays, same uniforms - so the result is the fp32 engine's, bit
    for bit, and later calls stay there without another detour."""
    G = _gpu()
    c = Case("bunny")
    render, cam = G.build_render(c, "auto"), G.build_camera(c)
    with torch.no_grad():
        render.network_fine.layers_col[0].weight.mul_(1e5)  # colour trunk only: densities / weights stay sane
    uv = c.t("uv").to(G.DEV)
    u = (c.t("u_coarse").to(G.DEV), c.t("u_fine").to(G.DEV))
    assert render.network_fine.resolved_engine() == "tc"
    with torch.no_grad():
        with pytest.warns(RuntimeWarning, match="fp16 range"):
            out = render.render_rays(uv, cam, uniforms=u)
        assert render.network_fine.resolved_engine() == "fp32"
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter("error", RuntimeWarning)  # no second detour
            again = render.render_rays(uv, cam, uniforms=u)
            img = render.render_image(40, 30, cam, ["color", "depth"], 1, 512)
        render.set_engine("fp32")
        ref = render.render_rays(uv, cam, uniforms=u)
        for k in ref:
            assert torch.equal(out[k], ref[k]) and torch.equal(again[k], ref[k]), k
        assert bool(torch.isfinite(ref["color"]).all()) and bool(torch.isfinite(img["color"]).all())
        assert float(ref["color"].abs().max()) > 1e3  # the blown-up colour trunk really is out of fp16 territory
        for engine in ("tc", "tc2"):
            render.set_engine(engine)
            with pytest.raises(FloatingPointError, match="65504"):
                render.render_rays(uv, cam, uniforms=u)
        # the image path of a fresh "auto" renderer takes the same detour once
        render.set_engine("auto")
        with pytest.warns(RuntimeWarning, match="fp16 range"):
            img2 = render.render_image(40, 30, cam, ["color", "depth"], 1, 512)
        assert bool(torch.isfinite(img2["color"]).all()) and render.network_fine.resolved_engine() == "fp32"
