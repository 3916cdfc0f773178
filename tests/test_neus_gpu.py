"""NeuS field variant on the GPU (csrc/neus_simt.cu behind neddf_b200.NeuS) against goldens recorded from the REAL
reference (tests/golden/make_neus_golden.py: the reference's NeuS inside its NeRFRender, grad mode) and the oracle
restatement: per-sample sdf / density / colour with explicit samples and with the fused ray geometry, the normal
against the oracle's gradient, render_rays through NeRFRender with the recorded uniforms, the image path (which the
reference cannot run for this network: its autograd.grad needs grad mode, render_image disables it)."""
import numpy as np
import pytest
import torch

from oracle import neddf_oracle as orc
from tests.helpers import PARITY_TOL, check_neus_normal, nerr
from tests.test_neus_oracle import NeusCase

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def build(c: NeusCase):
    import neddf_b200
    render = neddf_b200.NeRFRender(network_config=dict(c.net_cfg), **c.render_cfg)
    sd = {}
    for tag in ("fine", "coarse"):
        pre = f"w_{tag}." if f"w_{tag}.layers_sdf.0.weight" in c.z else "w_fine."
        for k, v in c.z.items():
            if k.startswith(pre):
                sd[f"network_{tag}." + k[len(pre):]] = torch.from_numpy(v)
    missing = render.load_state_dict(sd)
    assert not missing.missing_keys and not missing.unexpected_keys, missing  # the reference's state_dict layout
    render.to(DEV)
    render.set_iter(-1)
    cam = neddf_b200.Camera.from_matrix(neddf_b200.PinholeCalib(c.z["cam_calib"]), c.z["cam_R"], c.z["cam_T"]).to(DEV)
    cam.update_transform()
    return render, cam


def check_normal(c: NeusCase, tag: str, pos, got, ref, what):
    check_neus_normal(c.params(tag, torch.float64), c.nc, pos, got, ref, f"{tag} / {what}")


@pytest.mark.parametrize("name", ["relu", "tanhexp"])
def test_neus_field_matches_reference(name):
    import neddf_b200
    c = NeusCase(name)
    render, _ = build(c)
    d, o = orc.make_rays(c.t("uv"), c.cam)
    radius = neddf_b200.ray.CONE_RAY_RADIUS if c.rc.sampling_type == "cone" else 0.0
    for tag, net, dists in (("coarse", render.network_coarse, orc.coarse_dists(c.rc, c.t("u_coarse"))),
                            ("fine", render.network_fine, c.t("dists_fine"))):
        pos, dd, var = orc.make_samples(c.rc, d, o, dists)
        with torch.no_grad():
            out = net(neddf_b200.Sampling(pos.to(DEV), dd.contiguous().to(DEV), var.to(DEV)), with_normal=True)
            fused = net.forward_rays(d.to(DEV), o.to(DEV), dists.to(DEV), c.rc.sampling_type, radius, with_normal=True)
            plain = net(neddf_b200.Sampling(pos.to(DEV), dd.contiguous().to(DEV), var.to(DEV)))
        assert sorted(plain.keys()) == ["color", "density", "sdf"]  # the reference's dictionary (neus.py:155-160)
        assert torch.equal(plain["color"], out["color"])
        for k in ("sdf", "density"):  # continuous across the ReLU kinks: strict bound
            ref = c.z[f"field_{tag}_{k}"]
            assert out[k].shape == ref.shape
            assert nerr(out[k].cpu().numpy(), ref) < PARITY_TOL, (tag, k)
            assert nerr(fused[k].cpu().numpy(), ref) < PARITY_TOL, (tag, k, "fused geometry")
        for what, got in (("explicit samples", out["color"]), ("fused geometry", fused["color"])):
            check_normal(c, tag, pos, got.cpu().numpy(), c.z[f"field_{tag}_color"], "color, " + what)
        grad = orc.neus_forward(c.params(tag), c.nc, pos, dd)["gradients"].numpy()  # torch.autograd.grad, neus.py:133-142
        for what, got in (("explicit samples", out["normal"]), ("fused geometry", fused["normal"])):
            check_normal(c, tag, pos, got.cpu().numpy(), grad, what)


@pytest.mark.parametrize("name", ["relu", "tanhexp"])
def test_neus_render_rays_matches_reference(name):
    c = NeusCase(name)
    render, cam = build(c)
    with torch.no_grad():
        out = render.render_rays(c.t("uv").to(DEV), cam, uniforms=(c.t("u_coarse").to(DEV), c.t("u_fine").to(DEV)))
    ref_keys = sorted(k[4:] for k in c.z if k.startswith("out_"))
    assert sorted(out.keys()) == ref_keys  # no penalty keys for this variant (nerf_render.py:149-187)
    for k in ref_keys:
        tol = 1e-3 if k.startswith("weight") else PARITY_TOL  # same bounds as the NeDDF render test
        assert nerr(out[k].cpu().numpy(), c.z["out_" + k]) < tol, k


def test_neus_image_path_and_ragged_tiles():
    """render_image through the NeuS kernel (sample counts that are not multiples of the 64-sample tile or the
    16-sample sub-tile) against the oracle field on the same samples; training-mode calls are refused."""
    import neddf_b200
    c = NeusCase("tanhexp")
    render, cam = build(c)
    img = render.render_image(40, 30, cam, ["color", "depth", "transmittance"], 1, 333)
    assert img["color"].shape == (30, 40, 3) and bool(torch.isfinite(img["color"]).all())
    assert float(img["transmittance"].min()) >= 0.0 and float(img["transmittance"].max()) <= 1.0 + 1e-6
    net = render.network_fine
    g = torch.Generator().manual_seed(5)
    for n in (1, 15, 17, 63, 65, 1000, 148 * 64 + 5):
        pos = (torch.rand(1, n, 3, generator=g) * 2 - 1)
        dd = torch.nn.functional.normalize(torch.randn(1, n, 3, generator=g), dim=-1)
        with torch.no_grad():
            out = net(neddf_b200.Sampling(pos.to(DEV), dd.to(DEV), torch.zeros(1, n, 3, device=DEV)), with_normal=True)
        ref = orc.neus_forward(c.params("fine"), c.nc, pos, dd)
        for k, rk in (("sdf", "sdf"), ("density", "density"), ("color", "color"), ("normal", "gradients")):
            a, r = out[k].cpu().numpy(), ref[rk].numpy()
            assert np.abs(a - r).max() <= PARITY_TOL * max(np.abs(r).max(), 1.0), (n, k)
    with pytest.raises(NotImplementedError):
        render.render_rays(c.t("uv").to(DEV), cam)  # autograd enabled, trainable parameters
    # a parameter update is picked up by the next call (the packed copy is keyed on the tensors' version counters)
    pos = torch.rand(1, 40, 3, generator=g) * 2 - 1
    dd = torch.nn.functional.normalize(torch.randn(1, 40, 3, generator=g), dim=-1)
    s = neddf_b200.Sampling(pos.to(DEV), dd.to(DEV), torch.zeros(1, 40, 3, device=DEV))
    with torch.no_grad():
        before = net(s)["density"].clone()
        net.variance.mul_(1.5)
        after = net(s)["density"]
    P = c.params("fine")
    P["variance"] = P["variance"] * 1.5
    ref = orc.neus_forward(P, c.nc, pos, dd)["density"].numpy()
    assert nerr(after.cpu().numpy(), ref) < PARITY_TOL and float((after - before).abs().max()) > 1e-3
