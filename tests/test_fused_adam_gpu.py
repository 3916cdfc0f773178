"""GPU: the fused Adam step (neddf_field_adam_step, csrc/train_glue.cu) and FusedAdam on hardware.

- The kernel through the C ABI against an fp64 statement of torch.optim.Adam, at tensor counts on both sides of its
  32-tensor batches, sizes on both sides of one grid-stride pass (32 blocks x 256 threads = 8192 elements), and the
  hyperparameters and step counts a training run reaches; zero, underflowing, overflowing and non-finite gradients
  against torch's own fp32 Adam on the device.
- Refused calls change nothing and launch nothing.
- FusedAdam over NeDDF, NeRF and NeuS networks against torch.optim.Adam, with every kernel handle checked to have
  re-packed the stepped weights (bit-identical to a fresh network loaded from the state dict).
- The benchmark's training step, four steps in, against an fp64 Adam fed the same gradients, and against the oracle's
  gradients at the stepped weights.
Worst errors print with -s (``FUSED_ADAM_ERR`` lines), in units of u = 2^-24."""
import ctypes as C
import json
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import neddf_oracle as orc  # noqa: E402
from tests import field_configs as fcfg  # noqa: E402
from tests import nerf_neus_configs as ncfg  # noqa: E402
from tests.helpers import Case, nerr  # noqa: E402

DEV = torch.device("cuda:0")
U = 2.0 ** -24
K = 8  # per step: |x - x64| <= K u (|x64| + |x64 - x_before|)
GRAD_TOL = 1e-4
NUMELS = (0, 1, 255, 8191, 8192, 8193)
BIG = 3_000_017
HYPER = {  # lr, betas, eps, weight_decay
    "bench": (5e-4, (0.9, 0.999), 1e-8, 0.0),
    "decay": (5e-4, (0.9, 0.999), 1e-8, 1e-2),
    "beta1_0": (1e-3, (0.0, 0.5), 1e-8, 0.0),
    "betas_low": (1e-3, (0.5, 0.9), 1e-8, 1e-2),
    "eps_tiny": (5e-4, (0.9, 0.999), 1e-12, 0.0),
    "eps_big": (5e-4, (0.9, 0.999), 1e-3, 1e-2),
}
STEPS = (1, 2, 17, 10 ** 4, 10 ** 7)
# launches of one FusedAdam step on the golden training render (26 tensors): one Adam launch and the 4 of the re-pack,
# the same as before per-parameter step counts (measured on an H100 at both)
STEP_LAUNCHES = 5


def _report(**kw):
    print("FUSED_ADAM_ERR " + json.dumps(kw))


def _lib():
    from neddf_b200 import _lib as L
    return L, L.lib()


def _call(ps, gs, ms, vs, lr, betas, eps, wd, step, f=None, n=None, numel=None, null=None):
    """neddf_field_adam_step on lists of tensors; ``null`` = (array index 0..3, tensor index) passed as NULL."""
    L, lib = _lib()
    n = len(ps) if n is None else n
    cap = max(n, len(ps), 1)
    arrs = []
    for a, ts in enumerate((ps, gs, ms, vs)):
        ptrs = [t.data_ptr() for t in ts] + [0] * (cap - len(ts))
        if null is not None and null[0] == a:
            ptrs[null[1]] = None
        arrs.append((C.c_void_p * cap)(*ptrs))
    nums = [t.numel() for t in ps] + [0] * (cap - len(ps)) if numel is None else numel
    return lib.neddf_field_adam_step(f, *arrs, (C.c_int64 * cap)(*nums), n, lr, betas[0], betas[1], eps, wd, step,
                                     L.stream_ptr(DEV))


def _logu(n, lo, hi, g, signed=True):
    """fp32 values log-uniform in magnitude over [lo, hi], random signs."""
    x = torch.exp(torch.empty(n, dtype=torch.float64).uniform_(math.log(lo), math.log(hi), generator=g))
    if signed:
        x = x * (torch.randint(0, 2, (n,), generator=g) * 2 - 1)
    return x.float()


def _sizes(n, g):
    if n == 1:
        return [8193]
    sizes = [NUMELS[i % len(NUMELS)] for i in range(n)]
    sizes[int(torch.randint(0, n, (1,), generator=g))] = BIG
    return sizes


def _adam64(p, g, m, v, lr, betas, eps, wd, step):
    """torch.optim.Adam (foreach=False) in fp64 on fp64 inputs; eps and weight_decay are fp32 scalars in torch's fp32
    ops, so they are here."""
    b1, b2 = betas
    eps, wd = float(np.float32(eps)), float(np.float32(wd))
    if wd != 0.0:
        g = g + wd * p
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    p = p - lr / bc1 * m / (v.sqrt() / math.sqrt(bc2) + eps)
    return p, m, v


def _ulps(x, ref, before, floor=0.0):
    """max |x - ref| / (u (|ref| + |ref - before| + floor)); 0 / 0 counts as 0.  For parameters ``floor`` is the step
    size lr / (1 - b1^t): where exp_avg = b1 m + (1 - b1) g cancels, the update keeps the rounding of its terms."""
    x, ref, before = x.double(), ref.double(), before.double()
    den = U * (ref.abs() + (ref - before).abs() + floor)
    err = (x - ref).abs()
    assert bool(torch.isfinite(x).all()), "non-finite result"
    assert bool((err[den == 0] == 0).all())
    return float((err / den.clamp_min(1e-300))[den > 0].max()) if bool((den > 0).any()) else 0.0


@pytest.mark.parametrize("step", STEPS)
@pytest.mark.parametrize("hyper", list(HYPER))
def test_kernel_matches_fp64_adam(hyper, step):
    """Tensor counts 1, 31, 32, 33, 64 of mixed sizes (0 .. 3e6 elements) at one hyperparameter set and step count;
    gradients log-uniform in magnitude over [1e-12, 1e3] with random signs; moments of a run in progress (zero at step
    1).  Every element of p, exp_avg and exp_avg_sq within K u of the fp64 statement, relative to its value plus its
    change."""
    lr, betas, eps, wd = HYPER[hyper]
    g = torch.Generator().manual_seed(1000 * list(HYPER).index(hyper) + STEPS.index(step))
    worst = {"p": 0.0, "m": 0.0, "v": 0.0}
    for n in (1, 31, 32, 33, 64):
        sizes = _sizes(n, g)
        host = []
        for s in sizes:
            p = torch.randn(s, generator=g)
            gr = _logu(s, 1e-12, 1e3, g)
            m = torch.zeros(s) if step == 1 else _logu(s, 1e-12, 1e2, g)
            v = torch.zeros(s) if step == 1 else _logu(s, 1e-24, 1e4, g, signed=False)
            host.append((p, gr, m, v))
        dev = [[t.to(DEV) for t in ts] for ts in host]
        ps, gs, ms, vs = (list(x) for x in zip(*dev))
        assert _call(ps, gs, ms, vs, lr, betas, eps, wd, step) == 0
        torch.cuda.synchronize()
        for (p, gr, m, v), (pd, _, md, vd) in zip(host, dev):
            rp, rm, rv = _adam64(p.double().to(DEV), gr.double().to(DEV), m.double().to(DEV), v.double().to(DEV),
                                 lr, betas, eps, wd, step)
            if p.numel() == 0:
                continue
            worst["p"] = max(worst["p"], _ulps(pd, rp, p.to(DEV), lr / (1 - betas[0] ** step)))
            worst["m"] = max(worst["m"], _ulps(md, rm, m.to(DEV)))
            worst["v"] = max(worst["v"], _ulps(vd, rv, v.to(DEV)))
        assert max(worst.values()) <= K, (n, worst)
    _report(test="kernel", hyper=hyper, step=step, **{k + "_u": round(e, 2) for k, e in worst.items()})


@pytest.mark.parametrize("wd", [0.0, 1e-2])
def test_kernel_outside_fp32_range_matches_torch(wd):
    """Gradients of 0, of 1e-30 (g^2 underflows), large enough that g^2 or (1 - b2) g^2 overflows, NaN and +-inf:
    against torch.optim.Adam's fp32 step on the device over two steps - the same NaN and inf positions, finite values
    within K u."""
    g = torch.Generator().manual_seed(77)
    # (1e21: g^2 and (1 - b2) g g both overflow, whichever product comes first)
    special = torch.tensor([0.0, -0.0, 1e-30, -1e-30, 2e21, 1e21, -1e25, 3e38, float("nan"), float("inf"), -float("inf")])
    n = 8192 + 5
    grads = [torch.cat([special, torch.randn(n - special.numel(), generator=g)]) for _ in range(2)]
    grads[1][:special.numel()] = special.flip(0)
    p0 = torch.randn(n, generator=g).to(DEV)
    ref = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=1e-3, weight_decay=wd, foreach=False)
    p, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    worst = 0.0
    for it, gr in enumerate(grads):
        st = opt.state.get(ref, {})
        prev = [ref.detach().clone()] + [st[k].clone() if st else torch.zeros_like(p0) for k in ("exp_avg", "exp_avg_sq")]
        ref.grad = gr.to(DEV)
        opt.step()
        assert _call([p], [gr.to(DEV)], [m], [v], 1e-3, (0.9, 0.999), 1e-8, wd, it + 1) == 0
        torch.cuda.synchronize()
        st = opt.state[ref]
        for got, exp, pv, fl in zip((p, m, v), (ref.detach(), st["exp_avg"], st["exp_avg_sq"]), prev,
                                    (1e-3 / (1 - 0.9 ** (it + 1)), 0.0, 0.0)):
            assert torch.equal(torch.isnan(got), torch.isnan(exp)), it
            inf = torch.isinf(exp)
            assert torch.equal(torch.isinf(got), inf) and torch.equal(got[inf], exp[inf]), it
            fin = torch.isfinite(exp)
            worst = max(worst, _ulps(got[fin], exp[fin], pv[fin], fl))
        assert worst <= K, (it, worst)
    assert bool(torch.isnan(p[8:9]).all()) and bool(torch.isnan(p[9:11]).all())  # NaN and +-inf gradients poison p
    _report(test="outside_fp32", wd=wd, worst_u=round(worst, 2))


REFUSALS = (["n_tensors 0", "n_tensors 65", "step 0", "negative numel"] +
            [f"NULL {a} at {i}" for i in (0, 31, 40) for a in ("param", "grad", "exp_avg", "exp_avg_sq")] +
            ["field handle, 2 tensors short"])


@pytest.mark.parametrize("case", REFUSALS)
def test_refused_call_changes_nothing(case):
    """Every refusal happens before the first launch: NEDDF_E_INVALID, every tensor bit-identical, no launch counted.
    (A NULL in the second 32-tensor batch, a negative size or a handle whose layer count does not match the tensors
    must not leave the first batch stepped.)"""
    import neddf_b200
    L, lib = _lib()
    g = torch.Generator().manual_seed(5)
    net, f = None, None
    if case.startswith("field handle"):
        net = neddf_b200.NeDDF(**fcfg.kwargs("C1_default"))
        net.load_state_dict(fcfg.params("C1_default"))
        net.to(DEV)
        f = net._field(DEV)
        ps = [t for l in net._ordered_layers() for t in (l.weight, l.bias)][:-2]
        ps = [t.detach() for t in ps]
    else:
        # no empty tensor: its NULL storage would be refused in the first batch for the wrong reason
        ps = [torch.randn(s or 3, generator=g).to(DEV) for s in (_sizes(65, g) if case == "n_tensors 65" else _sizes(48, g))]
    gs = [torch.randn(t.shape, generator=g).to(DEV) for t in ps]
    ms = [torch.randn(t.shape, generator=g).to(DEV) for t in ps]
    vs = [torch.rand(t.shape, generator=g).to(DEV) for t in ps]
    snap = [t.clone() for t in ps + gs + ms + vs]
    kw = dict(lr=1e-2, betas=(0.9, 0.999), eps=1e-8, wd=0.0, step=3, f=f)
    if case == "n_tensors 0":
        kw["n"] = 0
    elif case == "step 0":
        kw["step"] = 0
    elif case == "negative numel":
        kw["numel"] = [t.numel() for t in ps]
        kw["numel"][40] = -1
    elif case.startswith("NULL"):
        _, a, _, i = case.split()
        kw["null"] = (("param", "grad", "exp_avg", "exp_avg_sq").index(a), int(i))
    torch.cuda.synchronize()
    launches = lib.neddf_launch_count()
    assert _call(ps, gs, ms, vs, **kw) == -1, case
    torch.cuda.synchronize()
    assert lib.neddf_launch_count() == launches
    for i, (a, b) in enumerate(zip(ps + gs + ms + vs, snap)):
        assert torch.equal(a, b), (case, i)
    if net is not None:
        net._release()


def _twin_check_nerf_neus(name, net, fresh, rays):
    """The next forward (and, with training kernels, the next training backward's parameter gradients) of ``net`` and of
    ``fresh`` (loaded from net's state dict) bit-identical: both kernel handles hold the stepped weights."""
    d, o, dists = rays
    kw = {"with_normal": True} if ncfg.variant(name) == "neus" else {}
    with torch.no_grad():
        a = net.forward_rays(d, o, dists, "cone", orc.CONE_RAY_RADIUS, **kw)
        b = fresh.forward_rays(d, o, dists, "cone", orc.CONE_RAY_RADIUS, **kw)
    for k in a:
        assert torch.equal(a[k], b[k]), (name, "forward", k)
    grads = []
    for m in (net, fresh):
        out = m.forward_rays(d, o, dists, "cone", orc.CONE_RAY_RADIUS, **kw)
        m.zero_grad(set_to_none=True)
        (out["density"].sum() + out["color"].sum() + (out["sdf"].sum() if "sdf" in out else 0)).backward()
        grads.append({k: p.grad.clone() for k, p in m.named_parameters()})
    for k in grads[0]:
        assert torch.equal(grads[0][k], grads[1][k]), (name, "grad", k)


def _build(kind, name):
    import neddf_b200
    if kind == "neddf":
        net = neddf_b200.NeDDF(**fcfg.kwargs(name))
        net.load_state_dict(fcfg.params(name))
        net.set_iter(fcfg.CONFIGS[name]["iter"])
    else:
        net = (neddf_b200.NeRF if ncfg.variant(name) == "nerf" else neddf_b200.NeuS)(**ncfg.kwargs(name))
        net.load_state_dict(ncfg.state_dict(name))
        net.set_iter(ncfg.CONFIGS[name]["iter"])
        net.training_kernels = True
    return net.to(DEV)


@pytest.mark.parametrize("kind,name", [("neddf", "C1_default"), ("neddf", "C7_deepest"), ("nerf", "N2_max_embed"),
                                       ("nerf", "N4_deep_train"), ("neus", "S2_max_embed"), ("neus", "S3_deepest")])
def test_fused_adam_repacks_every_handle(kind, name):
    """FusedAdam against torch.optim.Adam on one network over 3 steps (C1_default: 34 tensors, one handle call across
    the 32-tensor batch; C7_deepest: 54).  After each step the next forward - and for NeRF / NeuS the next training
    backward, which runs on the second handle - is bit-identical to a fresh network's loaded from the state dict."""
    from neddf_b200 import optim
    net, ref = _build(kind, name), _build(kind, name)
    fo = optim.FusedAdam(net.parameters(), lr=1e-3, weight_decay=1e-3, networks=[net])
    ro = torch.optim.Adam(ref.parameters(), lr=1e-3, weight_decay=1e-3, foreach=False)
    L, lib = _lib()
    g = torch.Generator().manual_seed(3)
    rays = tuple(t.to(DEV) for t in (fcfg.rays(7, 19, 4) if kind == "neddf" else ncfg.rays(7, 19, 4)))
    d, o, dists = rays
    n_tensors = 2 * len(net._ordered_layers())
    worst = 0.0
    for it in range(3):
        for a, b in zip(net.parameters(), ref.parameters()):
            gr = torch.randn(a.shape, generator=g).to(DEV)
            a.grad, b.grad = gr.clone(), gr.clone()
        before = [p.detach().clone() for p in ref.parameters()]
        torch.cuda.synchronize()
        launches = lib.neddf_launch_count()
        fo.step()
        ro.step()
        torch.cuda.synchronize()
        if kind == "neddf":  # one call: a launch per 32 tensors, then the re-pack
            assert lib.neddf_launch_count() - launches > (n_tensors + 31) // 32
        for a, b, b0 in zip(net.parameters(), ref.parameters(), before):
            worst = max(worst, _ulps(a.detach(), b.detach(), b0, 1e-3 / (1 - 0.9 ** (it + 1))))
        assert worst <= K, (it, worst)
        fresh = _build(kind, name)
        fresh.load_state_dict(net.state_dict())
        if kind == "neddf":
            net.zero_grad(set_to_none=True)
            with torch.no_grad():
                a = net.forward_rays(d, o, dists, "cone", orc.CONE_RAY_RADIUS)
                b = fresh.forward_rays(d, o, dists, "cone", orc.CONE_RAY_RADIUS)
            for k in a:
                assert torch.equal(a[k], b[k]), (it, k)
        else:
            _twin_check_nerf_neus(name, net, fresh, rays)
        fresh._release()
    _report(test="repack", config=name, tensors=n_tensors, worst_u=round(worst, 2))


def _render_step(render, cam, uv, u, tgt):
    """render_rays with fixed uniforms, RenderLoss, backward: (outputs, gradients by parameter name)."""
    from neddf_b200 import losses
    out = render.render_rays(uv, cam, uniforms=u)
    loss = torch.sum(torch.stack(list(losses.RenderLoss()(out, tgt).values())))
    render.zero_grad(set_to_none=True)
    loss.backward()
    return ({k: v.detach().clone() for k, v in out.items() if isinstance(v, torch.Tensor)},
            {k: p.grad.detach().clone() for k, p in render.named_parameters()})


@pytest.mark.parametrize("engine", ["fp32", "tc", "tc2"])
def test_training_step_several_steps_in(engine):
    """The benchmark's training step on the golden training render, 4 steps of render_rays (fixed uniforms), RenderLoss,
    backward, FusedAdam and ExponentialLR, beside an fp64 torch.optim.Adam fed the GPU's own gradients:
    - the parameters within the kernel bound times the step count;
    - the render and the gradients bit-identical to a fresh render's loaded from the state dict (no stale packed weights);
    - fp32 engine, 64 rays: gradients of the reference objective against fp64 autograd through the oracle at the stepped
      weights, within the end-to-end bound of the golden test (2 GRAD_TOL);
    - the launches of one optimiser step: one per 32 tensors plus one re-pack, as before per-parameter step counts."""
    import bench
    from neddf_b200 import optim
    from tests import gpu_util as Gu
    L, lib = _lib()
    c = Case("train")
    cam = Gu.build_camera(c)
    uv = c.t("uv").to(DEV)
    u = (c.t("u_coarse").to(DEV), c.t("u_fine").to(DEV))
    g = torch.Generator().manual_seed(12)
    tgt = {"color": torch.rand(uv.shape[0], 3, generator=g).to(DEV),
           "mask": (torch.rand(uv.shape[0], generator=g) > 0.3).float().to(DEV)}
    render = Gu.build_render(c, engine)
    opt = optim.FusedAdam.for_render(render, lr=5e-4)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, 0.5)
    names = [k for k, _ in render.named_parameters()]
    p64 = [p.detach().cpu().double().requires_grad_(True) for p in render.parameters()]
    o64 = torch.optim.Adam(p64, lr=5e-4, foreach=False)
    s64 = torch.optim.lr_scheduler.ExponentialLR(o64, 0.5)
    net = render.network_fine
    n_tensors = 2 * len(net._ordered_layers())
    # one re-pack on its own (after the handle's first pack), for the launch count of a step
    layers = net._ordered_layers()
    ws = (C.c_void_p * len(layers))(*[l.weight.data_ptr() for l in layers])
    bs = (C.c_void_p * len(layers))(*[l.bias.data_ptr() for l in layers])
    h = net._field(DEV)
    torch.cuda.synchronize()
    l0 = lib.neddf_launch_count()
    L.check(lib.neddf_field_set_weights(h, ws, bs, len(layers), L.stream_ptr(DEV)), "set_weights")
    repack = lib.neddf_launch_count() - l0
    sub = torch.arange(0, uv.shape[0], max(1, uv.shape[0] // 64))[:64]
    worst, worst_oracle, step_launches = 0.0, 0.0, None
    for it in range(4):
        _render_step(render, cam, uv, u, tgt)
        for a, b in zip(render.parameters(), p64):
            b.grad = a.grad.detach().cpu().double()
        torch.cuda.synchronize()
        l0 = lib.neddf_launch_count()
        opt.step()
        torch.cuda.synchronize()
        launches = lib.neddf_launch_count() - l0
        assert launches == (n_tensors + 31) // 32 + repack == STEP_LAUNCHES, (launches, repack)
        step_launches = launches
        before = [b.detach().clone() for b in p64]
        o64.step()
        sched.step()
        s64.step()
        for name, a, b, b0 in zip(names, render.parameters(), p64, before):
            e = _ulps(a.detach().cpu(), b.detach(), b0, 5e-4 / (1 - 0.9 ** (it + 1)))
            worst = max(worst, e)
            assert e <= K * (it + 1), (it, name, e)
        fresh = Gu.build_render(c, engine)
        fresh.load_state_dict(render.state_dict())
        out_a, grad_a = _render_step(render, cam, uv, u, tgt)
        out_b, grad_b = _render_step(fresh, cam, uv, u, tgt)
        for k in out_a:
            assert torch.equal(out_a[k], out_b[k]), (it, k)
        for k in grad_a:
            assert torch.equal(grad_a[k], grad_b[k]), (it, k)
        fresh.network_fine._release()
        if engine == "fp32":
            worst_oracle = max(worst_oracle, _oracle_grads(render, c, cam, uv, u, tgt, sub, bench))
    _report(test="train_steps", engine=engine, worst_u=round(worst, 2), oracle_grad_nerr=worst_oracle,
            step_launches=step_launches, tensors=n_tensors)


def _oracle_grads(render, c, cam, uv, u, tgt, sub, bench):
    """nerr of the GPU's gradients of bench.train_loss on the rays ``sub`` against fp64 autograd through the oracle, at
    the render's current weights; asserted below 2 GRAD_TOL (the golden end-to-end bound)."""
    out = render.render_rays(uv[sub], cam, uniforms=(u[0][sub], u[1][sub]))
    loss = bench.train_loss(out, tgt["color"][sub], tgt["mask"][sub])
    render.zero_grad(set_to_none=True)
    loss.backward()
    prefix = "network_fine."
    P = {k[len(prefix):]: p.detach().cpu().double().requires_grad_(True) for k, p in render.named_parameters()
         if k.startswith(prefix)}
    ref = orc.render_rays(P, P, c.fc, c.st, c.rc, uv[sub].cpu(), c.cam, u[0][sub].cpu().double(), u[1][sub].cpu().double(),
                          dtype=torch.float64)
    bench.train_loss(ref, tgt["color"][sub].cpu().double(), tgt["mask"][sub].cpu().double()).backward()
    worst = 0.0
    for k, p in render.named_parameters():
        e = nerr(p.grad.cpu().numpy(), P[k[len(prefix):]].grad.numpy())
        assert e < 2 * GRAD_TOL, (k, e)
        worst = max(worst, e)
    return worst
