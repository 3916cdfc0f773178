"""NeuS training backward on the GPU (csrc/neus_train.cu + neddf_wgrad behind neddf_b200.NeuS with training_kernels=True).

Ordered so that a miss says where it is: (a) the kernel's buffers against the per-layer quantities of the fp64
restatement (tests/neus_train_oracle.py), (b) neddf_wgrad on exactly those buffers against an fp64 matmul of the same
buffers (and on gradient-sized operands), (c) field-level parameter gradients from the recorded upstream gradients of
the REAL reference (tests/golden/make_neus_train_golden.py), (d) render_rays end to end with the recorded objective,
(e) upstream gradients on sdf / normal, (f) ragged sample counts, (g) determinism."""
import pytest
import torch

from oracle import neddf_oracle as orc
from tests import neus_train_oracle as nto
from tests.helpers import nerr
from tests.test_neus_train_emul import BUF_NAMES, TrainCase, buffer_shapes, compare, oracle_grads

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def small_net(act="tanhExp", seed=5):
    import neddf_b200
    torch.manual_seed(seed)
    net = neddf_b200.NeuS(embed_pos_rank=4, embed_dir_rank=2, sdf_layer_count=3, col_layer_count=2, activation_type=act,
                          init_variance=0.4, skips=[0])
    with torch.no_grad():
        net.layers_sdf[-1].weight[0].mul_(6.0)
        net.layers_sdf[-1].bias[0].add_(0.35)
    net.training_kernels = True
    return net.to(DEV)


def oracle_params(net, dtype=torch.float64):
    names = [n for n, _, _ in orc.neus_layer_shapes(orc.NeusConfig(**net_kw(net)))]
    layers = net._ordered_layers()
    return nto.params_from_torch([l.weight.detach().cpu() for l in layers], [l.bias.detach().cpu() for l in layers], names,
                                 net.variance.detach().cpu(), dtype), names


def net_kw(net):
    return dict(embed_pos_rank=net.embed_pos_rank, embed_dir_rank=net.embed_dir_rank, sdf_layer_count=net.sdf_layer_count,
                col_layer_count=net.col_layer_count, activation_type=net.activation_type, skips=list(net.skips))


def random_samples(n, seed):
    g = torch.Generator().manual_seed(seed)
    pos = (torch.rand(1, n, 3, generator=g) * 2 - 1) * 0.7
    dd = torch.nn.functional.normalize(torch.randn(1, n, 3, generator=g), dim=-1)
    ups = {"sdf": torch.randn(1, n, generator=g), "density": torch.randn(1, n, generator=g),
           "color": torch.randn(1, n, 3, generator=g), "normal": torch.randn(1, n, 3, generator=g)}
    return pos, dd, ups


def kernel_buffers(net, pos, dd, ups):
    """One neddf_neus_train_backward call; its nine buffers on the host."""
    import ctypes as C

    from neddf_b200 import _lib as L
    nc = orc.NeusConfig(**net_kw(net))
    n = pos.shape[1]
    buf = {k: torch.full(s, float("nan"), device=DEV) for k, s in buffer_shapes(nc, n).items()}
    bufs = (C.c_void_p * 9)(*[buf[k].data_ptr() for k in BUF_NAMES])
    h = net._train_field(DEV)
    d = {k: v.to(DEV).contiguous() for k, v in ups.items()}
    pos_d, dd_d = pos.to(DEV).contiguous(), dd.to(DEV).contiguous()  # alive until the kernel has run
    L.check(L.lib().neddf_neus_train_backward(h, L.ptr(pos_d), L.ptr(dd_d), n, L.ptr(d["sdf"]),
                                              L.ptr(d["density"]), L.ptr(d["color"]), L.ptr(d["normal"]), bufs, L.stream_ptr(DEV)),
            "neus_train_backward")
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in buf.items()}


def fp64_reference(net, pos, dd, ups):
    P, names = oracle_params(net)
    out, t = nto.neus_train_forward_jac(P, orc.NeusConfig(**net_kw(net)), pos.double(), dd.double(), keep=True)
    sum(((out[k] * ups[k].double()).sum() for k in ("sdf", "density", "color", "normal"))).backward()
    return P, names, t


def test_a_kernel_buffers_match_the_per_layer_oracle():
    """One 64-sample tile: E4, the SDF layer outputs XS and pre-activation gradients GS (value + Jacobian rows), the
    colour activations XC and pre-activation gradients GC, the head gradient, the per-sample variance terms."""
    net = small_net()
    pos, dd, ups = random_samples(64, 1)
    buf = kernel_buffers(net, pos, dd, ups)
    P, _, t = fp64_reference(net, pos, dd, ups)
    E4 = torch.cat([t["E"][:, None, :], t["EJ"]], 1)
    assert nerr(buf["E4"].numpy(), E4.detach().numpy()) < 1e-5, "E4"
    for l in range(net.sdf_layer_count):
        gs = torch.cat([t["sdf_z"][l].grad[:, None, :], t["sdf_Jz"][l].grad], 1).numpy()
        assert nerr(buf["GS"][l].numpy(), gs) < 2e-5, ("GS", l, nerr(buf["GS"][l].numpy(), gs))
        if l < net.sdf_layer_count - 1:
            xs = torch.cat([t["sdf_y"][l][:, None, :], t["sdf_Jy"][l]], 1).detach().numpy()
            assert nerr(buf["XS"][l].numpy(), xs) < 2e-5, ("XS", l)
    assert nerr(buf["XC0"].numpy(), t["X0"].detach().numpy()) < 2e-5, "XC0"
    assert nerr(buf["FO"].numpy(), t["F"].detach().numpy()) < 2e-5, "FO"
    for l in range(net.col_layer_count):
        assert nerr(buf["XC"][l].numpy(), t["col_h"][l].detach().numpy()) < 2e-5, ("XC", l)
        assert nerr(buf["GC"][l].numpy(), t["col_z"][l].grad.numpy()) < 2e-5, ("GC", l)
    assert nerr(buf["GH"].numpy(), t["zh"].grad.numpy()) < 2e-5, "GH"
    assert abs(float(buf["GV"].double().sum()) - float(P["variance"].grad)) <= 2e-5 * max(1.0, abs(float(P["variance"].grad)))


def _wgrad(A, lda, col0, ka, B, rows):
    from neddf_b200 import _lib as L
    lib = L.lib()
    out = torch.full((ka, 256), float("nan"), device=DEV)
    ws = torch.empty(int(lib.neddf_wgrad_workspace_bytes()) // 4, device=DEV)
    L.check(lib.neddf_wgrad(L.ptr(A), lda, col0, ka, L.ptr(B), 256, rows, L.ptr(out), 256, 256, L.ptr(ws), L.stream_ptr(DEV)), "wgrad")
    torch.cuda.synchronize()
    return out.cpu().double()


def test_b_wgrad_on_the_kernel_buffers():
    """neddf_wgrad on the very buffers of (a) - 4-row SDF operands, the E4 / XC0 heads with unaligned widths, the
    3-column head gradient - against an fp64 matmul of the same buffers."""
    net = small_net()
    pos, dd, ups = random_samples(64, 1)
    buf = kernel_buffers(net, pos, dd, ups)
    n = 64
    cases = [(buf["E4"].reshape(4 * n, -1), buf["GS"][0].reshape(4 * n, 256)),
             (buf["XS"][0].reshape(4 * n, 256), buf["GS"][1].reshape(4 * n, 256)),
             (buf["XC0"], buf["GC"][0]), (buf["FO"], buf["GC"][0]), (buf["GH"], buf["XC"][-1])]
    for A, B in cases:
        lda = A.shape[1]
        for c0 in range(0, lda, 128):
            ka = min(128, lda - c0)
            got = _wgrad(A.to(DEV).contiguous(), lda, c0, ka, B.to(DEV).contiguous(), A.shape[0])
            ref = A[:, c0:c0 + ka].double().t() @ B.double()
            assert float((got - ref).abs().max() / ref.abs().max()) < 1e-5, (tuple(A.shape), c0)


def test_b_wgrad_keeps_precision_on_gradient_sized_operands():
    """Gradients of a loss averaged over many rays are 1e-5 .. 1e-8: in plain fp16 hi / lo operands they are subnormal
    and lose up to a few 1e-3; the per-column power-of-two scaling of neddf_wgrad keeps them at fp32 accuracy."""
    g = torch.Generator().manual_seed(4)
    rows = 4 * 2000
    A = torch.randn(rows, 100, generator=g) * torch.logspace(-3, 0, 100)
    B = torch.randn(rows, 256, generator=g) * 1e-7
    B[:, :64] *= 1e-3
    got = _wgrad(A.to(DEV), 100, 0, 100, B.to(DEV), rows)
    ref = A.double().t() @ B.double()
    assert float((got - ref).abs().max() / ref.abs().max()) < 1e-5
    got = _wgrad(B.to(DEV), 256, 0, 64, A.to(DEV).repeat(1, 3)[:, :256].contiguous(), rows)  # tiny A columns too
    ref = B[:, :64].double().t() @ A.repeat(1, 3)[:, :256].double()
    assert float((got - ref).abs().max() / ref.abs().max()) < 1e-5


def build_render(c: TrainCase):
    import neddf_b200
    render = neddf_b200.NeRFRender(network_config=dict(c.net_cfg), **c.render_cfg)
    sd = {}
    for tag in ("fine", "coarse"):
        for k, v in c.state_dict(tag).items():
            sd[f"network_{tag}.{k}"] = torch.from_numpy(v)
    res = render.load_state_dict(sd)
    assert not res.missing_keys and not res.unexpected_keys, res
    render.to(DEV)
    render.set_iter(-1)
    for net in (render.network_coarse, render.network_fine):
        net.training_kernels = True
    cam = neddf_b200.Camera.from_matrix(neddf_b200.PinholeCalib(c.z["cam_calib"]), c.z["cam_R"], c.z["cam_T"]).to(DEV)
    cam.update_transform()
    return render, cam


def render_grads(render, c: TrainCase):
    grads = {}
    for n, p in render.named_parameters():
        if p.grad is not None:
            grads[n] = grads.get(n, 0) + p.grad.detach().cpu().numpy()
    return grads


@pytest.mark.parametrize("name", ["relu", "tanhexp"])
@pytest.mark.parametrize("fused", [True, False])
def test_c_field_gradients_match_the_reference(name, fused):
    """The recorded upstream gradients into forward_rays (fused geometry) / forward(Sampling); parameter gradients
    against the REAL reference's to 1e-4 (ReLU: the kinked rule of helpers.assert_parity)."""
    import neddf_b200
    c = TrainCase(name)
    render, _ = build_render(c)
    d, o, passes = c.passes()
    radius = neddf_b200.ray.CONE_RAY_RADIUS if c.rc.sampling_type == "cone" else 0.0
    render.zero_grad()
    loss = 0
    for tag, dists in passes:
        net = getattr(render, "network_" + tag)
        if fused:
            out = net.forward_rays(d.to(DEV), o.to(DEV), dists.to(DEV), c.rc.sampling_type, radius)
        else:
            pos, dd, var = orc.make_samples(c.rc, d, o, dists)
            out = net(neddf_b200.Sampling(pos.to(DEV), dd.contiguous().to(DEV), var.to(DEV)))
        loss = loss + (out["density"] * c.t(f"up_{tag}_density").to(DEV)).sum() + (out["color"] * c.t(f"up_{tag}_color").to(DEV)).sum()
    loss.backward()
    grads = {}
    for tag in ("coarse", "fine"):
        net = getattr(render, "network_" + tag)
        for k, p in net.named_parameters():
            grads[f"network_{c.net_tag(tag)}.{k}"] = p.grad.detach().cpu().numpy()
    compare(c, grads, oracle_grads(c, torch.float64))


def objective(out, tc, tm):
    """config/loss/nerf_loss.yaml: ColorLoss (1.0, coarse 0.1) + MaskBCELoss (0.05, coarse 0.005), nerf_trainer.py:118-121."""
    total = 0.0
    for suffix, wc, wm in (("", 1.0, 0.05), ("_coarse", 0.1, 0.005)):
        total = total + wc * torch.mean(torch.square(out["color" + suffix] - tc))
        m = torch.clamp(1.0 - out["transmittance" + suffix], 1e-6, 1.0 - 1e-6)
        total = total + wm * -torch.mean(tm * torch.log(m) + (1.0 - tm) * torch.log(1.0 - m))
    return total


@pytest.mark.parametrize("name", ["relu", "tanhexp"])
def test_d_render_rays_trains_end_to_end(name):
    """render_rays under autograd with the recorded uniforms and objective: loss to 1e-4, gradients to 2e-4 (ReLU:
    the kinked rule - here the rays come from this package's camera, which may differ from the reference's in the
    last bit)."""
    c = TrainCase(name)
    render, cam = build_render(c)
    render.zero_grad()
    out = render.render_rays(c.t("uv").to(DEV), cam, uniforms=(c.t("u_coarse").to(DEV), c.t("u_fine").to(DEV)))
    loss = objective(out, c.t("target_color").to(DEV), c.t("target_mask").to(DEV))
    assert abs(float(loss.detach()) - float(c.z["loss"])) <= 1e-4 * abs(float(c.z["loss"]))
    loss.backward()
    compare(c, render_grads(render, c), tol=2e-4)


def test_e_sdf_and_normal_gradients_against_fp64():
    """Upstream gradients on the returned sdf and normal (with_normal=True) reach the parameters as in fp64 autograd."""
    import neddf_b200
    net = small_net()
    pos, dd, ups = random_samples(200, 2)
    out = net(neddf_b200.Sampling(pos.to(DEV), dd.to(DEV), torch.zeros(1, 200, 3, device=DEV)), with_normal=True)
    assert all(out[k].requires_grad for k in ("sdf", "density", "color", "normal"))
    sum((out[k] * ups[k].to(DEV)).sum() for k in ("sdf", "density", "color", "normal")).backward()
    P, names, _ = fp64_reference(net, pos, dd, ups)
    for l, name in zip(net._ordered_layers(), names):
        for what, p in (("weight", l.weight), ("bias", l.bias)):
            ref = P[f"{name}.{what}"].grad.numpy()
            ref = ref.T if what == "weight" else ref
            assert nerr(p.grad.cpu().numpy(), ref) < 5e-5, (name, what)
    assert abs(float(net.variance.grad) - float(P["variance"].grad)) <= 5e-5 * abs(float(P["variance"].grad))


@pytest.mark.parametrize("n", [1, 63, 65, 148 * 64 + 5])
def test_f_ragged_sample_counts(n):
    import neddf_b200
    net = small_net()
    pos, dd, ups = random_samples(n, 3)
    out = net(neddf_b200.Sampling(pos.to(DEV), dd.to(DEV), torch.zeros(1, n, 3, device=DEV)))
    ((out["density"] * ups["density"].to(DEV)).sum() + (out["color"] * ups["color"].to(DEV)).sum()).backward()
    ups = dict(ups, sdf=torch.zeros_like(ups["sdf"]), normal=torch.zeros_like(ups["normal"]))
    P, names, _ = fp64_reference(net, pos, dd, ups)
    for l, name in zip(net._ordered_layers(), names):
        ref = P[f"{name}.weight"].grad.numpy().T
        assert nerr(l.weight.grad.cpu().numpy(), ref) < 5e-5, (n, name)
        assert nerr(l.bias.grad.cpu().numpy(), P[f"{name}.bias"].grad.numpy()) < 5e-5, (n, name)
    assert abs(float(net.variance.grad) - float(P["variance"].grad)) <= 5e-5 * max(1e-3, abs(float(P["variance"].grad)))


def test_g_two_backward_calls_are_bitwise_equal():
    import neddf_b200
    net = small_net("ReLU")
    pos, dd, ups = random_samples(3000, 4)
    s = neddf_b200.Sampling(pos.to(DEV), dd.to(DEV), torch.zeros(1, 3000, 3, device=DEV))
    got = []
    for _ in range(2):
        net.zero_grad()
        out = net(s)
        ((out["density"] * ups["density"].to(DEV)).sum() + (out["color"] * ups["color"].to(DEV)).sum()).backward()
        got.append([p.grad.clone() for p in net.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*got))


def test_default_still_refuses_autograd():
    c = TrainCase("tanhexp")
    render, cam = build_render(c)
    for net in (render.network_coarse, render.network_fine):
        net.training_kernels = False
    with pytest.raises(NotImplementedError, match="forward-only"):
        render.render_rays(c.t("uv").to(DEV), cam)
