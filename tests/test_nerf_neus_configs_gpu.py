"""GPU: the NeRF and NeuS kernels and their training backward at every structure of tests/nerf_neus_configs.py, against
the fp64 oracle - forward through every entry point at ragged and multi-wave sample counts, parameter gradients through
both autograd entry points, the training handle's refusal past its depth, and bitwise repeatability of the training
backward (NeRF, NeuS and the NeDDF training step) over a caching allocator primed with NaN and with zeros, which shows
any element read before a kernel wrote it."""
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import neddf_oracle as orc  # noqa: E402
from tests import nerf_neus_configs as ncfg  # noqa: E402
from tests import neus_train_oracle as nto  # noqa: E402
from tests.helpers import PARITY_TOL, Case, assert_parity, check_neus_normal, nerr  # noqa: E402

DEV = torch.device("cuda:0")
GRAD_TOL = 1e-4
# S5's variance gradient sums per-sample terms of both signs across a steep density (10 variance = 20): on the 64-sample
# ray path they cancel to -0.0052, and the fp32 restatement of the same graph (tests/neus_train_oracle.py in fp32) sits
# 4.7e-4 from fp64 there (3.5e-5 .. 1.7e-4 on the other three paths; the kernel measured 4.7e-4 on an H100)
GRAD_TOL_OVERRIDE = {("S5_sharp", "variance"): 1e-3}
# the 64-sample tile and its 16-sample sub-tiles from both sides, and 269 tiles: more than the H100's 132 SMs take at
# once, so the persistent CTAs loop
COUNTS = (1, 15, 16, 17, 63, 64, 65, 2 * 132 * 64 + 5)
RAY_SHAPES = ((1, 1), (1, 2), (1, 15), (1, 16), (1, 17), (3, 21), (4, 16), (5, 13), (131, 129))
GEOMETRY = (("point", 0.0), ("cone", orc.CONE_RAY_RADIUS))


def _report(**kw):
    """One line per entry (visible with pytest -s): the largest errors."""
    print("NERF_NEUS_CONFIG_ERR " + json.dumps(kw))


def _net(name, train=False):
    import neddf_b200
    net = (neddf_b200.NeRF if ncfg.variant(name) == "nerf" else neddf_b200.NeuS)(**ncfg.kwargs(name))
    net.load_state_dict(ncfg.state_dict(name))
    net.to(DEV)
    net.set_iter(ncfg.CONFIGS[name]["iter"])
    net.training_kernels = train
    return net


def _p64(name, requires_grad=False):
    return {k: v.double().requires_grad_(requires_grad) for k, v in ncfg.params(name).items()}


def _ray_samples(kind, d, o, dists):
    """Sample geometry in fp32, one rounding per operation like the kernels' prologue: at rank 10 the encoding
    multiplies positions by 2^9, so positions computed in fp64 would not be the ones the kernel evaluates."""
    if kind == "point":
        return orc.point_samples(d, o, dists)
    return orc.cone_samples(d, o, dists, orc.CONE_RAY_RADIUS)


def _oracle(name, P, pos, dirs, var):
    """fp64 outputs; NeuS's 'normal' is the reverse-mode gradient of the sdf (neus.py:133-142)."""
    cfg = ncfg.config(name)
    if ncfg.variant(name) == "nerf":
        with torch.no_grad():
            return orc.nerf_forward(P, cfg, ncfg.lowpass_alpha(name), pos.double(), dirs.double(), var.double())
    out = orc.neus_forward(P, cfg, pos.double(), dirs.double())
    out["normal"] = out.pop("gradients")
    return out


def _compare(name, P, pos, got, ref, what):
    """Largest error per key; NeuS colour and normal with the kink witness of check_neus_normal."""
    worst = {}
    for k in ref:
        a, r = got[k].detach().cpu().numpy(), ref[k].detach().numpy()
        if k in ("color", "normal") and ncfg.variant(name) == "neus":
            worst[k] = check_neus_normal(P, ncfg.config(name), pos, a, r, f"{name} {what}:{k}")
        else:
            assert_parity(a, r, PARITY_TOL, ncfg.kinked(name), f"{name} {what}:{k}")
            worst[k] = nerr(a, r)
    return worst


def _check_sharp_density(name, P, out, ref_sdf):
    """S5: where the sdf is past 5.25 exp(-20 sdf) is below half fp32's smallest subnormal, so the density is exactly 0;
    everywhere the density matches the op-by-op fp32 restatement of the kernel's own sdf."""
    sdf = out["sdf"].cpu()
    dens = out["density"].cpu()
    past = ref_sdf > 5.25
    assert bool(torch.isfinite(dens).all())
    assert torch.equal(dens[past], torch.zeros_like(dens[past]))
    ref32 = orc.neus_density(sdf, P["variance"].float())
    differ = (dens == 0) != (ref32 == 0)  # the two exp implementations may round the last subnormal differently
    assert bool((torch.maximum(dens, ref32)[differ] < 1e-37).all())
    assert nerr(dens.numpy(), ref32.numpy()) < 1e-6
    return int(past.sum())


def _merge(worst, tag, errs):
    for k, e in errs.items():
        worst[f"{tag}_{k}"] = max(worst.get(f"{tag}_{k}", 0.0), e)


@pytest.mark.parametrize("name", ncfg.NAMES)
def test_forward_matches_oracle(name):
    """forward(Sampling) and forward_rays with point and cone geometry at every count of COUNTS; NeuS also with
    with_normal=True (sdf, density and colour bit-identical to the call without it)."""
    import neddf_b200
    net = _net(name)
    P = _p64(name)
    neus = ncfg.variant(name) == "neus"
    sharp = ncfg.CONFIGS[name].get("sharpen", False)
    worst, underflows = {}, 0

    def run(call, ref, pos, tag):
        nonlocal underflows
        with torch.no_grad():
            out = call(with_normal=True) if neus else call()
            if neus:
                plain = call()
                for k in ("sdf", "density", "color"):
                    assert torch.equal(plain[k], out[k]), (tag, k)
        _merge(worst, tag, _compare(name, P, pos, out, ref, f"{tag} n={pos.shape[0] * pos.shape[1]}"))
        if sharp:
            underflows += _check_sharp_density(name, P, out, ref["sdf"].float())

    for n in COUNTS:
        pos, dirs, var = ncfg.samples(1, n, ncfg.SEED[name] + 10 + n)
        s = neddf_b200.Sampling(pos.to(DEV), dirs.to(DEV), var.to(DEV))
        run(lambda **kw: net(s, **kw), _oracle(name, P, pos, dirs, var), pos, "sampling")
    for B, S in RAY_SHAPES:
        d, o, dists = ncfg.rays(B, S, ncfg.SEED[name] + 20 + B * S)
        dd, od, distsd = d.to(DEV), o.to(DEV), dists.to(DEV)
        for kind, radius in GEOMETRY:
            if kind == "cone" and S == 1:
                continue  # a frustum ends at the next edge: a cone ray needs two
            pos, dirs, var = _ray_samples(kind, d, o, dists)
            run(lambda **kw: net.forward_rays(dd, od, distsd, kind, radius, **kw), _oracle(name, P, pos, dirs, var), pos, kind)
    torch.cuda.synchronize()
    if sharp:
        assert underflows > 1000, underflows
        worst["density_underflows"] = underflows
    _report(test="forward", config=name, **worst)


def _upstream(name, B, S, seed):
    g = torch.Generator().manual_seed(seed)
    up = {"density": torch.randn(B, S, generator=g), "color": torch.randn(B, S, 3, generator=g)}
    if ncfg.variant(name) == "neus":
        up.update(sdf=torch.randn(B, S, generator=g), normal=torch.randn(B, S, 3, generator=g))
    return up


def _fp64_grads(name, pos, dirs, var, up):
    """Parameter gradients of sum(out * up) by fp64 autograd through the oracle, in the modules' layout."""
    P = _p64(name, requires_grad=True)
    cfg = ncfg.config(name)
    if ncfg.variant(name) == "nerf":
        out = orc.nerf_forward(P, cfg, ncfg.lowpass_alpha(name), pos.double(), dirs.double(), var.double())
    else:  # the kernel's forward-mode formulation of the reference's graph (tests/test_neus_train_emul.py pins the two)
        out = nto.neus_train_forward_jac(P, cfg, pos.double(), dirs.double())
    sum((out[k] * up[k].double()).sum() for k in up).backward()
    return {k: (v.grad.t() if k.endswith(".weight") else v.grad) for k, v in P.items()}


def _module_grads(net, call, up):
    out = call()
    net.zero_grad(set_to_none=True)
    sum((out[k] * up[k].to(DEV)).sum() for k in up).backward()
    return {k: p.grad.detach().clone() for k, p in net.named_parameters()}


def _training_paths(name, net):
    """(tag, call, fp32 samples, (B, S)): forward_rays with cone geometry and forward(Sampling), each at a ragged count
    and at one full 64-sample tile."""
    import neddf_b200
    kw = {"with_normal": True} if ncfg.variant(name) == "neus" else {}
    paths = []
    for B, S in ((5, 13), (2, 32)):
        d, o, dists = ncfg.rays(B, S, ncfg.SEED[name] + 40 + B)
        call = (lambda d=d, o=o, dists=dists: net.forward_rays(d.to(DEV), o.to(DEV), dists.to(DEV), "cone",
                                                               orc.CONE_RAY_RADIUS, **kw))
        paths.append((f"rays{B * S}", call, _ray_samples("cone", d, o, dists), (B, S)))
    for n in (65, 64):
        pos, dirs, var = ncfg.samples(1, n, ncfg.SEED[name] + 50 + n)
        call = (lambda pos=pos, dirs=dirs, var=var: net(neddf_b200.Sampling(pos.to(DEV), dirs.to(DEV), var.to(DEV)), **kw))
        paths.append((f"sampling{n}", call, (pos, dirs, var), (1, n)))
    return paths


@pytest.mark.parametrize("name", ncfg.TRAIN)
def test_training_gradients_match_autograd(name):
    """training_kernels=True: random upstream gradients on density and colour (NeuS: sdf and normal too) through
    forward_rays and forward(Sampling); every parameter gradient (and NeuS's variance) against fp64 autograd through the
    oracle - 1e-4 for tanhExp, the kinked rule of helpers.assert_parity for ReLU / LeakyReLU."""
    net = _net(name, train=True)
    worst = {}
    for tag, call, (pos, dirs, var), (B, S) in _training_paths(name, net):
        up = _upstream(name, B, S, ncfg.SEED[name] + 60 + B * S)
        ref = _fp64_grads(name, pos, dirs, var, up)
        got = _module_grads(net, call, up)
        assert set(got) == set(ref)
        e_max = 0.0
        for k, r in ref.items():
            a, r = got[k].cpu().numpy(), r.numpy()
            assert a.shape == r.shape, k
            assert np.isfinite(a).all(), (tag, k)
            if ncfg.kinked(name) and a.ndim > 0:
                assert_parity(a, r, GRAD_TOL, True, f"{name} {tag}:{k}")
            else:
                assert nerr(a, r) < GRAD_TOL_OVERRIDE.get((name, k), GRAD_TOL), (tag, k, nerr(a, r))
            e_max = max(e_max, nerr(a, r))
        worst[tag] = e_max
    _report(test="training", config=name, **worst)


def test_training_handle_refuses_past_its_depth():
    """13 layers run forward, but the training backward takes 2..12: under autograd with training_kernels=True the call
    raises a RuntimeError naming the limit, and no parameter receives a gradient."""
    net = _net("N3_deep_fwd", train=True)
    d, o, dists = ncfg.rays(3, 21, 5)
    with pytest.raises(RuntimeError, match=r"2\.\.12"):
        out = net.forward_rays(d.to(DEV), o.to(DEV), dists.to(DEV), "cone", orc.CONE_RAY_RADIUS)
        (out["density"].sum() + out["color"].sum()).backward()
    assert all(p.grad is None for p in net.parameters())
    torch.cuda.synchronize()


def _prime_allocator(value):
    """Hand the caching allocator free blocks filled with ``value`` in both of its pools (blocks up to 1 MB come from
    2 MB segments, larger ones are split from the 512 MB blocks), so that buffers torch.empty returns next hold it."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    blocks = [torch.full((1 << 27,), value, device=DEV) for _ in range(4)]
    blocks += [torch.full((n,), value, device=DEV) for n in (1 << 17, 1 << 15, 1 << 12, 1 << 8) for _ in range(64)]
    torch.cuda.synchronize()
    del blocks
    for n in (1 << 10, 1 << 22):  # the priming took: fresh buffers from both pools hold the value
        probe = torch.empty(n, device=DEV)
        assert bool(torch.isnan(probe).all()) if value != value else bool((probe == value).all()), n
        del probe


def _poisoned_and_clean(step):
    """``step()`` (a dict of tensors) once after NaN-filled and once after zero-filled blocks: both finite and equal."""
    runs = []
    for value in (float("nan"), 0.0):
        _prime_allocator(value)
        runs.append({k: v.detach().cpu() for k, v in step().items()})
    for k in runs[0]:
        assert bool(torch.isfinite(runs[0][k]).all()) and bool(torch.isfinite(runs[1][k]).all()), k
        assert torch.equal(runs[0][k], runs[1][k]), (k, float((runs[0][k] - runs[1][k]).abs().max()))
    return len(runs[0])


@pytest.mark.parametrize("name", ["N2_max_embed", "N6_warmup", "S2_max_embed", "S4_eight_skips"])
def test_training_backward_is_bitwise_repeatable(name):
    """One tanhExp and one ReLU entry per variant, 3,008 samples over several CTAs, forward + backward twice over
    differently poisoned memory: no buffer element is read before it is written."""
    neus = ncfg.variant(name) == "neus"
    d, o, dists = ncfg.rays(47, 64, ncfg.SEED[name] + 70)
    up = _upstream(name, 47, 64, ncfg.SEED[name] + 71)

    def step():
        net = _net(name, train=True)
        return _module_grads(net, lambda: net.forward_rays(d.to(DEV), o.to(DEV), dists.to(DEV), "cone", orc.CONE_RAY_RADIUS,
                                                           **({"with_normal": True} if neus else {})), up)

    _report(test="repeatable", config=name, tensors=_poisoned_and_clean(step))


@pytest.mark.parametrize("engine", ["fp32", "tc", "tc2"])
def test_neddf_training_step_is_bitwise_repeatable(engine):
    """The NeDDF training step of the benchmark - render_rays with fixed uniforms, RenderLoss, backward, one FusedAdam
    step - on the golden training render, twice over differently poisoned memory: parameter gradients and updated
    parameters bit-identical."""
    from neddf_b200 import losses, optim
    from tests import gpu_util as G
    c = Case("train")
    uv = c.t("uv").to(DEV)
    u = (c.t("u_coarse").to(DEV), c.t("u_fine").to(DEV))
    g = torch.Generator().manual_seed(11)
    tgt = {"color": torch.rand(uv.shape[0], 3, generator=g).to(DEV),
           "mask": (torch.rand(uv.shape[0], generator=g) > 0.3).float().to(DEV)}

    def step():
        render, cam = G.build_render(c, engine), G.build_camera(c)
        opt = optim.FusedAdam.for_render(render, lr=5e-4)
        out = render.render_rays(uv, cam, uniforms=u)
        loss = torch.sum(torch.stack(list(losses.RenderLoss()(out, tgt).values())))
        opt.zero_grad(set_to_none=True)
        loss.backward()
        res = {"loss": loss.detach()}
        res.update({"grad:" + k: p.grad.detach().clone() for k, p in render.named_parameters()})
        opt.step()
        res.update({"param:" + k: p.detach().clone() for k, p in render.named_parameters()})
        return res

    _report(test="neddf_repeatable", engine=engine, tensors=_poisoned_and_clean(step))
