"""GPU: the NeDDF field engines and the training backward at every structure of tests/field_configs.py, against the
fp64 oracle - forward through every entry point, ragged and multi-wave sample counts, parameter gradients, engine
resolution at the tensor-core bounds, and the weight-gradient GEMM at the shapes these structures produce."""
import json
from functools import lru_cache

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import neddf_oracle as orc  # noqa: E402
from tests import field_configs as fcfg  # noqa: E402
from tests.helpers import PARITY_TOL, assert_parity, nerr  # noqa: E402

DEV = torch.device("cuda:0")
GRAD_TOL = 1e-4  # the bar of test_gpu_parity.test_field_backward_matches_autograd
OUT_KEYS = ("distance", "density", "color", "fields_penalty", "aux_grad")
TC_PAIRS = [p for p in fcfg.PAIRS if p[1] != "fp32"]


def _report(**kw):
    """One line per measurement (visible with pytest -s): the largest errors per config and engine."""
    print("FIELD_CONFIG_ERR " + json.dumps(kw))


def _net(name, engine):
    import neddf_b200
    net = neddf_b200.NeDDF(**fcfg.kwargs(name))
    net.load_state_dict(fcfg.params(name))
    net.to(DEV)
    net.set_iter(fcfg.CONFIGS[name]["iter"])
    net.engine = engine
    return net


def _p64(name):
    return {k: v.double() for k, v in fcfg.params(name).items()}


def _oracle(name, pos, dirs, var, taps=None):
    with torch.no_grad():
        return orc.field_forward(_p64(name), fcfg.field_config(name), fcfg.state(name), pos.double(), dirs.double(),
                                 var.double(), taps=taps)


def _ray_samples(kind, d, o, dists):
    """Sample geometry in fp32, one rounding per operation like the reference's Ray (and the kernels' prologue):
    the positional encoding multiplies positions by up to 2^15 here, so positions computed in fp64 instead would
    differ from the kernels' by more than the parity bound at the high ranks; the network is then evaluated in fp64."""
    if kind == "point":
        return orc.point_samples(d, o, dists)
    return orc.cone_samples(d, o, dists, orc.CONE_RAY_RADIUS)


def _check_status(net, engine):
    if engine != "fp32":
        net.check_engine_status()  # FloatingPointError if an activation left fp16 range


def _compare(name, got, ref, keys, what):
    worst = 0.0
    for k in keys:
        a = got[k].detach().cpu().numpy()
        r = ref[k].detach().numpy()
        assert_parity(a, r, PARITY_TOL, fcfg.kinked(name), f"{what}:{k}")
        worst = max(worst, nerr(a, r))
    return worst


@pytest.mark.parametrize("name,engine", fcfg.PAIRS)
def test_forward_matches_oracle(name, engine):
    """Every forward entry point, n in {1, 31, 32, 33} (tc tiles 32 samples, fp32 16): Sampling tensors, fused point
    and cone geometry, the images-only program (need_penalty=False) and one full early-termination segment, which
    runs the images-only program and must agree with it bit for bit."""
    import neddf_b200
    net = _net(name, engine)
    worst = {}
    with torch.no_grad():
        for n in (1, 31, 32, 33):
            pos, dirs, var = fcfg.samples(1, n, fcfg.SEED[name] + 10 + n)
            out = net(neddf_b200.Sampling(pos.to(DEV), dirs.to(DEV), var.to(DEV)))
            e = _compare(name, out, _oracle(name, pos, dirs, var), OUT_KEYS, f"sampling n={n}")
            worst["sampling"] = max(worst.get("sampling", 0.0), e)
            _check_status(net, engine)
        for B, S in ((1, 2), (1, 31), (2, 16), (3, 11)):
            d, o, dists = fcfg.rays(B, S, fcfg.SEED[name] + 20 + B * S)
            dd, od, distsd = d.to(DEV), o.to(DEV), dists.to(DEV)
            for kind, radius in (("point", 0.0), ("cone", orc.CONE_RAY_RADIUS)):
                ref = _oracle(name, *_ray_samples(kind, d, o, dists))
                full = net.forward_rays(dd, od, distsd, kind, radius, need_penalty=True, need_aux=True)
                e = _compare(name, full, ref, OUT_KEYS, f"{kind} {B}x{S}")
                worst[kind] = max(worst.get(kind, 0.0), e)
                images = net.forward_rays(dd, od, distsd, kind, radius, need_penalty=False, need_aux=True)
                e = _compare(name, images, ref, ("distance", "density", "color", "aux_grad"), f"{kind} images {B}x{S}")
                worst["images"] = max(worst.get("images", 0.0), e)
                evals = net.forward_rays(dd, od, distsd, kind, radius, need_penalty=False, need_aux=False)
                density = torch.full((B, S), float("nan"), device=DEV)
                color = torch.full((B, S, 3), float("nan"), device=DEV)
                net.forward_rays_segment(dd, od, distsd, kind, radius, 0, S, None, None, density, color)
                assert torch.equal(density, evals["density"]) and torch.equal(color, evals["color"]), (kind, B, S)
                _check_status(net, engine)
    _report(test="forward", config=name, engine=engine, **worst)


@pytest.mark.parametrize("name,engine", [p for p in TC_PAIRS if p[0] in ("C1_default", "C2_minimal", "C7_deepest")])
def test_forward_with_more_tiles_than_ctas(name, engine):
    """2 * 132 * 32 + 5 samples: every CTA of the persistent tensor-core kernel takes several tiles, the last one
    ragged (weight ring carried across tiles)."""
    import neddf_b200
    net = _net(name, engine)
    n = 2 * 132 * 32 + 5
    pos, dirs, var = fcfg.samples(1, n, fcfg.SEED[name] + 30)
    with torch.no_grad():
        out = net(neddf_b200.Sampling(pos.to(DEV), dirs.to(DEV), var.to(DEV)))
    _check_status(net, engine)
    ref, kink = _oracle_cached(name, n)
    e = _compare(name, out, ref, OUT_KEYS, f"n={n}")
    # kinked configurations: every sample outside the parity bound must sit next to a kink (some hidden
    # pre-activation within KINK_WITNESS of 0), where fp32 evaluations legitimately take the other slope.  With 24
    # layers of 256 units most samples do (median distance ~2e-5), but the samples clear of every kink would expose a
    # tile or weight-ring fault, which corrupts whole tiles
    bad = torch.zeros(n, dtype=torch.bool)
    for k in OUT_KEYS:
        r = ref[k].reshape(n, -1)
        err = (out[k].cpu().double().reshape(n, -1) - r).abs() / r.abs().max()
        bad |= (err >= PARITY_TOL).any(1)
    worst_kink = float(kink[bad].max()) if bool(bad.any()) else 0.0
    _report(test="many_tiles", config=name, engine=engine, n=n, err=e, outliers=int(bad.sum()), outlier_kink=worst_kink,
            clear=int((kink >= KINK_WITNESS).sum()))
    assert worst_kink < KINK_WITNESS, (int(bad.sum()), worst_kink)


KINK_WITNESS = 1e-4  # |pre-activation| below which a sample counts as sitting on a kink


@lru_cache(maxsize=None)
def _oracle_cached(name, n):
    """fp64 outputs and, per sample, the smallest |pre-activation| over every hidden unit of every layer."""
    pos, dirs, var = fcfg.samples(1, n, fcfg.SEED[name] + 30)
    taps = {}
    ref = _oracle(name, pos, dirs, var, taps)
    pre = [v.abs().min(1).values for k, v in taps.items() if k.endswith("_pre") and k[:3] in ("ddf", "col")]
    return ref, torch.stack(pre, 1).min(1).values


def _train_step(net, call, g):
    out = call()
    loss = sum((out[k] * g[k].to(DEV)).sum() for k in ("density", "color", "fields_penalty"))
    net.zero_grad(set_to_none=True)
    loss.backward()
    return out, {k: p.grad.detach().clone() for k, p in net.named_parameters()}


@pytest.mark.parametrize("name,engine", fcfg.PAIRS)
def test_training_gradients_match_autograd(name, engine):
    """The training path (forward of the engine keeping pre-activations, field_bwd.cu, neddf_wgrad /
    neddf_colsum_value_rows) through forward_rays (cone geometry) and forward(Sampling), for random upstream
    gradients: every parameter gradient against fp64 autograd through the oracle, and a second run bit-identical."""
    import neddf_b200
    net = _net(name, engine)
    cfg, st = fcfg.field_config(name), fcfg.state(name)
    B, S = 3, 13
    d, o, dists = fcfg.rays(B, S, fcfg.SEED[name] + 40)
    sp, sd, sv = fcfg.samples(2, 20, fcfg.SEED[name] + 41)
    paths = {
        "rays": (lambda: net.forward_rays(d.to(DEV), o.to(DEV), dists.to(DEV), "cone", orc.CONE_RAY_RADIUS),
                 _ray_samples("cone", d, o, dists), (B, S)),
        "sampling": (lambda: net(neddf_b200.Sampling(sp.to(DEV), sd.to(DEV), sv.to(DEV))),
                     (sp, sd, sv), (2, 20)),
    }
    worst = {}
    for tag, (call, (pos, dirs, var), shape) in paths.items():
        gd, gc, gp = fcfg.upstream(*shape, fcfg.SEED[name] + 42)
        g = {"density": gd, "color": gc, "fields_penalty": gp}
        P = {k: v.clone().requires_grad_(True) for k, v in _p64(name).items()}
        ref = orc.field_forward(P, cfg, st, pos.double(), dirs.double().contiguous(), var.double())
        sum((ref[k] * g[k].double()).sum() for k in g).backward()
        out, grads = _train_step(net, call, g)
        _check_status(net, engine)
        worst[tag + "_fwd"] = _compare(name, out, ref, ("density", "color", "fields_penalty"), tag)
        e_max = 0.0
        for k, v in P.items():
            got = grads[k].cpu().numpy()
            assert got.shape == tuple(v.shape), k
            e = nerr(got, v.grad.numpy())
            assert e < GRAD_TOL, (tag, k, e)
            e_max = max(e_max, e)
        worst[tag + "_grad"] = e_max
        _, again = _train_step(net, call, g)
        for k in grads:
            assert torch.equal(grads[k], again[k]), (tag, k)  # fixed summation order
    _report(test="training", config=name, engine=engine, **worst)


@pytest.mark.parametrize("name", fcfg.NAMES)
def test_engine_resolution_at_the_tensor_core_bounds(name):
    """"auto" runs the tensor-core engine exactly where its AUX layout covers the inputs (n_e0 <= 64, off_h <= 96);
    past either bound it runs fp32 and an explicit "tc" / "tc2" is refused before any launch."""
    import neddf_b200
    net = _net(name, "auto")
    tc = "tc" in fcfg.CONFIGS[name]["engines"]
    assert net.resolved_engine() == ("tc" if tc else "fp32")
    pos, dirs, var = fcfg.samples(1, 5, 1)
    s = neddf_b200.Sampling(pos.to(DEV), dirs.to(DEV), var.to(DEV))
    for engine in ("tc", "tc2"):
        net.engine = engine
        if tc:
            assert net.resolved_engine() == engine
            continue
        with pytest.raises(RuntimeError, match="tensor-core"):
            net.resolved_engine()
        with pytest.raises(RuntimeError, match="tensor-core"), torch.no_grad():
            net(s)
    torch.cuda.synchronize()


def _wgrad(A, lda, col0, ka, Bm):
    from neddf_b200 import _lib as L
    rows = Bm.shape[0]
    out = torch.full((ka, 256), float("nan"), device=DEV)
    ws = torch.empty(int(L.lib().neddf_wgrad_workspace_bytes()) // 4, device=DEV)
    L.check(L.lib().neddf_wgrad(L.ptr(A), lda, col0, ka, L.ptr(Bm), 256, rows, L.ptr(out), 256, 256, L.ptr(ws),
                                L.stream_ptr(DEV)), "wgrad")
    torch.cuda.synchronize()
    return out.cpu().double()


@pytest.mark.parametrize("spread", [False, True])
@pytest.mark.parametrize("rows,lda,col0,ka", [(4 * 111, 195, 128, 67), (4 * 8453, 96, 0, 96)])
def test_wgrad_at_sweep_shapes(rows, lda, col0, ka, spread):
    """neddf_wgrad at the shapes of these structures: the colour input of C6 (lda 195, second 128-column tile of 67
    columns) and the colour input of C3 / a full 96-column tile over many rows.  With ``spread`` the operand columns
    span 1e-20 .. 1e3 (A) and 1e-8 .. 1e3 (B, which keeps every product inside fp32's normal range) with one all-zero
    column each - gradients of a loss averaged over rays sit far below fp16's range, which the GEMM's per-column
    power-of-two scaling must absorb.  Each element's error is normalised by sum_r |A[r,m] B[r,n]|, so a small column
    cannot hide behind a large one."""
    g = torch.Generator().manual_seed(rows + lda)
    A = torch.randn(rows, lda, generator=g)
    Bm = torch.randn(rows, 256, generator=g)
    if spread:
        A *= torch.logspace(-20, 3, lda, dtype=torch.float64)[torch.randperm(lda, generator=g)].float()
        Bm *= torch.logspace(-8, 3, 256, dtype=torch.float64)[torch.randperm(256, generator=g)].float()
        A[:, col0 + ka // 3] = 0.0
        Bm[:, 77] = 0.0
    out = _wgrad(A.to(DEV), lda, col0, ka, Bm.to(DEV))
    a = A[:, col0:col0 + ka].double()
    ref = a.t() @ Bm.double()
    den = a.abs().t() @ Bm.double().abs()
    assert torch.equal(out[den == 0], torch.zeros_like(out[den == 0]))
    e = float(((out - ref).abs()[den > 0] / den[den > 0]).max())
    _report(test="wgrad", rows=rows, lda=lda, col0=col0, ka=ka, spread=spread, err=e)
    assert e < 1e-5, e
