"""The kernels on either side of the field network, across every sample count and batch shape the renderer accepts:
coarse edges and sample geometry (csrc/geometry.cu), compositing and its backward, early ray termination
(csrc/composite.cu), hierarchical resampling (csrc/sample_pdf.cu) and the training objective (csrc/train_glue.cu).

Each kernel is called through the C ABI, so that every NULL-pointer combination is reachable, and compared with the
oracle twice: in fp32, the arithmetic the kernels restate, and in fp64 on the same inputs cast up, the arbiter.  The
bounds are tests.ray_cases.tol(kind, E); tests/test_ray_kernels_arbiter.py shows on the CPU that the fp32 oracle itself
needs that much.  Ray counts straddle the grid-stride passes of the kernels (64 rays per SM for compositing and
resampling, 1024 per SM for the termination kernel), edge counts the 32-sample blocks, the opt-in shared memory above
48 KB and the refusals above 200 KB.  Run with -s to see the largest error of each case."""
import itertools

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import neddf_oracle as orc  # noqa: E402
from tests import ray_cases as R  # noqa: E402
from tests.helpers import PARITY_TOL, Case, assert_parity, nerr  # noqa: E402

DEV = torch.device("cuda:0")
E_INVALID, E_UNSUPPORTED = -1, -3
SMALL_B = ["1", "7", "8", "9", "33"]
GRID_B = ["P-1", "P", "P+1"]  # P = 64 rays per SM: one grid-stride pass of compositing and resampling


def _L():
    from neddf_b200 import _lib as L
    return L


def _sm() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def n_rays(tok: str) -> int:
    """Ray count from a token: an integer, or an expression of P = 64 * SM count (Q = 1024 * SM count)."""
    return int(eval(tok, {"P": 64 * _sm(), "Q": 1024 * _sm()}))


def _call(fn, *args):
    """Call a C ABI entry on the current stream, raise like the library's callers, synchronise."""
    L = _L()
    L.check(getattr(L.lib(), fn)(*args, L.stream_ptr(DEV)), fn)
    torch.cuda.synchronize()


def _refused(code, fn, *args):
    with pytest.raises(RuntimeError, match=f"code {code}"):
        _call(fn, *args)


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _report(what, errs):
    print(f"[ray kernels] {what}: " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))


# ------------------------------------------------------------------------------------------------ compositing --

def _composite(dists, dens, col, pen, outs=("weight", "depth", "color", "transmittance", "fields_penalty"),
               status=None):
    """neddf_composite with only the outputs named in ``outs``; unwritten outputs stay NaN."""
    L = _L()
    B, E = dists.shape
    res = {"weight": _nan(B, E - 1), "depth": _nan(B), "color": _nan(B, 3), "transmittance": _nan(B),
           "fields_penalty": _nan(B)}
    res = {k: v for k, v in res.items() if k in outs}
    _call("neddf_composite", L.ptr(dists), L.ptr(dens), L.ptr(col), L.ptr(pen), B, E, R.MAX_DIST,
          L.ptr(res.get("weight")), L.ptr(res.get("depth")), L.ptr(res.get("color")), L.ptr(res.get("transmittance")),
          L.ptr(res.get("fields_penalty")), L.ptr(status))
    return res


def _composite_runs():
    runs = []
    for E in (1, 2, 3, 32, 33, 34, 65, 194, 258, 770, 1537, 3201, 5000):
        toks = SMALL_B if E <= 770 else ["1", "7", "33"]
        if E in (33, 194):
            toks = toks + GRID_B
        if E == 65:
            toks = toks + ["3*P+5"]
        runs.append((E, toks))
    return runs


@pytest.mark.parametrize("E,toks", _composite_runs())
def test_composite_forward(E, toks):
    """Every output against the fp32 and the fp64 oracle, for each density family; the penalty off leaves the other
    outputs bit for bit; empty space gives zero weights and colour and depth = T * max_dist exactly (T is not 1 but
    (1 + 1e-7)^(E-1): the reference adds 1e-7 to every factor).  E = 1 is a ray without intervals: T = 1."""
    worst = {"fp32": 0.0, "fp64": 0.0}
    bound = R.tol("composite", E)
    for tok, fam in itertools.product(toks, R.FAMILIES):
        B = n_rays(tok)
        d, s, c, p = R.ray_inputs(fam, B, E)
        dd, sd, cd, pd = (t.to(DEV) for t in (d, s, c, p))
        got = _composite(dd, sd, cd, pd)
        for tag, dtype in (("fp32", torch.float32), ("fp64", torch.float64)):
            ref = R.composite_ref(d, s, c, p, dtype)
            for k, v in ref.items():
                e = R.nerr64(got[k], v)
                worst[tag] = max(worst[tag], e)
                assert e < bound, (tok, fam, tag, k, e, bound)
        if fam == "zero" or E == 1:
            assert bool((got["depth"] == got["transmittance"] * R.MAX_DIST).all()), (tok, fam)
            assert bool((got["weight"] == 0.0).all()) and bool((got["color"] == 0.0).all()), (tok, fam)
            assert E > 1 or bool((got["transmittance"] == 1.0).all())
        off = _composite(dd, sd, cd, None, outs=("weight", "depth", "color", "transmittance"))
        for k, v in off.items():
            assert torch.equal(v, got[k]), (tok, fam, k)
    _report(f"composite E={E} (bound {bound:.1e})", worst)


@pytest.mark.parametrize("E,tok", [(33, "9"), (194, "P+1")])
def test_composite_null_outputs(E, tok):
    """Every allowed subset of NULL outputs (colour out needs colour in, penalty out needs penalty in): the outputs that
    remain are bitwise those of the full call.  The two forbidden combinations are refused."""
    L = _L()
    B = n_rays(tok)
    d, s, c, p = (t.to(DEV) for t in R.ray_inputs("translucent", B, E))
    full = _composite(d, s, c, p)
    names = list(full)
    for mask in range(1 << len(names)):
        outs = [k for i, k in enumerate(names) if mask >> i & 1]
        for with_c, with_p in itertools.product((True, False), repeat=2):
            if ("color" in outs and not with_c) or ("fields_penalty" in outs and not with_p):
                continue
            got = _composite(d, s, c if with_c else None, p if with_p else None, outs=outs)
            for k in outs:
                assert torch.equal(got[k], full[k]), (outs, with_c, with_p, k)
    w, o, po = _nan(B, E - 1), _nan(B, 3), _nan(B)
    _refused(E_INVALID, "neddf_composite", L.ptr(d), L.ptr(s), None, L.ptr(p), B, E, R.MAX_DIST, L.ptr(w), None,
             L.ptr(o), None, None, None)
    _refused(E_INVALID, "neddf_composite", L.ptr(d), L.ptr(s), L.ptr(c), None, B, E, R.MAX_DIST, L.ptr(w), None,
             None, None, L.ptr(po), None)
    assert bool(torch.isnan(w).all())


@pytest.mark.parametrize("E,tok", [(33, "9"), (194, "P+1")])
def test_composite_nan_flag(E, tok):
    """A NaN density on the last ray sets status bit 1 (check_status raises like the reference's assert); every other
    ray's outputs are unchanged."""
    import tests.gpu_util as G
    B = n_rays(tok)
    d, s, c, p = (t.to(DEV) for t in R.ray_inputs("translucent", B, E))
    clean = _composite(d, s, c, p)
    s_nan = s.clone()
    s_nan[B - 1, E // 2] = float("nan")
    status = torch.zeros(2, dtype=torch.int32, device=DEV)
    got = _composite(d, s_nan, c, p, status=status)
    assert int(status[0]) & 1
    for k in got:
        assert torch.equal(got[k][:B - 1], clean[k][:B - 1]), k
    assert bool(torch.isnan(got["weight"][B - 1, E // 2:]).all())
    render = G.build_render(Case("bunny"))
    render.integrate_volume_render(d, s_nan, c, p)
    with pytest.raises(AssertionError, match="NaN"):
        render.check_status()
    render.check_status()  # read and cleared


# --------------------------------------------------------------------------------------- compositing backward --

def _composite_backward(dists, dens, col, g, outs=("density", "color", "penalty")):
    """neddf_composite_backward; ``g`` maps output names to upstream gradients or None (NULL)."""
    L = _L()
    B, E = dists.shape
    res = {"density": _nan(B, E), "color": _nan(B, E, 3), "penalty": _nan(B, E)}
    res = {k: v for k, v in res.items() if k in outs}
    _call("neddf_composite_backward", L.ptr(dists), L.ptr(dens), L.ptr(col), B, E, R.MAX_DIST,
          L.ptr(g.get("weight")), L.ptr(g.get("depth")), L.ptr(g.get("color")), L.ptr(g.get("transmittance")),
          L.ptr(g.get("fields_penalty")), L.ptr(res.get("density")), L.ptr(res.get("color")),
          L.ptr(res.get("penalty")))
    return res


def _backward_runs():
    runs = []
    for E in (2, 3, 32, 33, 34, 65, 194, 258, 770, 1537, 3201):
        toks = SMALL_B if E <= 258 else ["1", "7", "33"]
        if E == 194:
            toks = toks + GRID_B
        if E == 65:
            toks = toks + ["3*P+5"]
        runs.append((E, toks))
    return runs


@pytest.mark.parametrize("E,toks", _backward_runs())
def test_composite_backward(E, toks):
    """Gradients of density, colour and penalty for random upstream gradients of all five outputs against autograd
    through the oracle in fp32 and in fp64; the closing edge gets exactly 0.  From E = 770 the backward's shared
    memory is above 48 KB; E = 3201 is its largest edge count."""
    worst = {"fp32": 0.0, "fp64": 0.0}
    bound = R.tol("composite_grad", E)
    for tok, fam in itertools.product(toks, R.FAMILIES):
        B = n_rays(tok)
        d, s, c, p = R.ray_inputs(fam, B, E)
        g = R.upstream(B, E)
        got = _composite_backward(d.to(DEV), s.to(DEV), c.to(DEV), {k: v.to(DEV) for k, v in g.items()})
        for tag, dtype in (("fp32", torch.float32), ("fp64", torch.float64)):
            ref = R.composite_grad_ref(d, s, c, p, g, dtype)
            for k, v in zip(("density", "color", "penalty"), ref):
                e = R.nerr64(got[k], v)
                worst[tag] = max(worst[tag], e)
                assert e < bound, (tok, fam, tag, k, e, bound)
        for k, v in got.items():
            assert bool((v[:, E - 1] == 0.0).all()), (tok, fam, k)  # the closing edge
    _report(f"composite backward E={E} (bound {bound:.1e})", worst)


@pytest.mark.parametrize("E,tok", [(33, "9"), (770, "P+1")])
def test_composite_backward_null_pointers(E, tok):
    """Each NULL upstream gradient is bitwise a zero-filled one; each NULL output leaves the others unchanged.
    E = 3202 needs more than 200 KB of shared memory and is refused on the host, before any launch."""
    L = _L()
    B = n_rays(tok)
    d, s, c, _ = (t.to(DEV) for t in R.ray_inputs("translucent", B, E))
    g = {k: v.to(DEV) for k, v in R.upstream(B, E).items()}
    full = _composite_backward(d, s, c, g)
    for k in g:
        zero = dict(g, **{k: torch.zeros_like(g[k])})
        null = {j: v for j, v in g.items() if j != k}
        a, b = _composite_backward(d, s, c, zero), _composite_backward(d, s, c, null)
        for j in a:
            assert torch.equal(a[j], b[j]), (k, j)
    for drop in full:
        got = _composite_backward(d, s, c, g, outs=[k for k in full if k != drop])
        for k, v in got.items():
            assert torch.equal(v, full[k]), (drop, k)
    E = 3202
    d, s, c, _ = (t.to(DEV) for t in R.ray_inputs("translucent", 1, E))
    gd = torch.zeros(1, device=DEV)
    out = _nan(1, E)
    _refused(E_UNSUPPORTED, "neddf_composite_backward", L.ptr(d), L.ptr(s), L.ptr(c), 1, E, R.MAX_DIST, None,
             L.ptr(gd), None, None, None, L.ptr(out), None, None)
    assert bool(torch.isnan(out).all())  # nothing ran


# ------------------------------------------------------------------------------------------------- resampling --

def _sample_pdf(dists, w, u, n_new, cat, status=None):
    """neddf_sample_pdf with the ids and the kernel's own cdf; ``w`` is sanitised in place."""
    L = _L()
    B, E = dists.shape
    out = _nan(B, (E if cat else 0) + n_new)
    ids = torch.full((B, n_new), -1, dtype=torch.int64, device=DEV)
    cdf = _nan(B, E)
    _call("neddf_sample_pdf", L.ptr(dists), L.ptr(w), L.ptr(u), B, E, n_new, 1 if cat else 0, L.ptr(out),
          L.ptr(ids) if n_new else None, L.ptr(cdf), L.ptr(status))
    return out, ids, cdf


def _exact_cdf(w, cat):
    """The kernel's cdf in exact arithmetic from its fp32 steps: sanitise, +1e-2, smoothing (cat_coarse=False), the
    fp32 pdf over the L1 norm summed exactly and rounded once, then the cumulative sum in fp64, rounded once."""
    b = orc.sanitise_weights(w) + 1e-2
    if not cat and b.shape[1] > 1:
        b = torch.cat([b[:, :1], 0.5 * (torch.maximum(b[:, 2:], b[:, 1:-1]) + torch.maximum(b[:, :-2], b[:, 1:-1])),
                       b[:, -1:]], 1)
    denom = b.abs().double().sum(1, keepdim=True).float().clamp_min(1e-12)
    pdf = b / denom
    return torch.cat([torch.zeros(b.shape[0], 1, dtype=torch.float64), torch.cumsum(pdf.double(), 1)], 1).float()


def _interpolate(dists, cdf, u):
    """base_neural_render.py:77-98 in fp32 torch ops on the CPU, from a given cdf: one rounding per operation, like the
    kernel's NS / NM / NA / __fdiv_rn."""
    ids = torch.searchsorted(cdf, u, right=True)
    below, above = (ids - 1).clamp_min(0), ids.clamp_max(cdf.shape[1] - 1)
    c0, c1 = cdf.gather(1, below), cdf.gather(1, above)
    d0, d1 = dists.gather(1, below), dists.gather(1, above)
    denom = c1 - c0
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)
    return d0 + ((u - c0) / denom) * (d1 - d0), ids


def _uniforms(B, F, seed, cdf=None, edges=True):
    """Uniforms with the edge values 0 and nextafter(1, 0) and, given a cdf, entries equal to cdf values (ties of the
    right-sided search)."""
    u = torch.rand(B, F, generator=torch.Generator().manual_seed(seed))
    if not edges:
        return u
    if F >= 1:
        u[:, 0] = 0.0
    if F >= 2:
        u[:, -1] = float(np.nextafter(np.float32(1), np.float32(0)))
    if cdf is not None and F >= 4:
        E = cdf.shape[1]
        u[:, 1], u[:, 2] = cdf[:, E // 2], cdf[:, 1]
    return u.contiguous()


PDF_SHAPES = [(2, 1, True), (2, 1, False), (3, 1, False), (33, 31, True), (33, 32, True), (33, 33, True),
              (33, 31, False), (33, 32, False), (33, 33, False), (65, 129, True), (65, 447, True), (65, 448, True),
              (65, 512, False), (65, 513, False), (1025, 1025, True), (2049, 2049, True)]


@pytest.mark.parametrize("E,F,cat", PDF_SHAPES)
def test_sample_pdf(E, F, cat):
    """The kernel's cdf is the exactly summed cdf of the fp32 pdf (a few ulp), monotone from 0; the ids are the
    right-sided search of the uniforms in that cdf, exactly; the samples are the fp32 interpolation from that cdf,
    merged and sorted, bit for bit; and the whole against the fp32 and the fp64 oracle.  Covers the 32-lane blocks,
    both sides of each power of two of the bitonic sort, the shared memory above 48 KB (E = 1025: 98,336 B) and near
    the 200 KB cap (E = 2049: 196,640 B); the weights are sanitised in place (negative -> -0.0, NaN -> 0)."""
    toks = ["1", "9", "P+1"] if E <= 1025 else ["7"]
    worst = {"cdf ulp": 0.0, "fp32": 0.0, "fp64": 0.0}
    bound = R.tol("sample_pdf", E)
    for tok, fam in itertools.product(toks, R.PDF_FAMILIES):
        B = n_rays(tok)
        d = R.ray_inputs("translucent", B, E)[0]
        w = R.pdf_weights(fam, B, E - 1)
        dd = d.to(DEV)
        for edges in (False, True):
            # uniforms at 0, at nextafter(1, 0) and equal to entries of the kernel's own cdf
            u = _uniforms(B, F, E, cdf if edges else None, edges)
            wd = w.to(DEV)
            status = torch.zeros(2, dtype=torch.int32, device=DEV)
            out, ids, cdf = _sample_pdf(dd, wd, u.to(DEV), F, cat, status)
            out, ids, cdf = out.cpu(), ids.cpu(), cdf.cpu()
            assert int(status[0]) == 0 and int(status[1]) == 0, (tok, fam)
            assert torch.equal(wd.cpu().view(torch.int32), orc.sanitise_weights(w).view(torch.int32)), (tok, fam)
            ex = _exact_cdf(w, cat)
            ulp = torch.from_numpy(np.spacing(np.abs(ex.numpy())))
            e_ulp = float(((cdf - ex).abs() / ulp).max())
            worst["cdf ulp"] = max(worst["cdf ulp"], e_ulp)
            assert e_ulp <= 4, (tok, fam, e_ulp)
            assert bool((cdf[:, 0] == 0).all()) and bool((cdf[:, 1:] >= cdf[:, :-1]).all()), (tok, fam)
            new, ids_ref = _interpolate(d, cdf, u)
            assert torch.equal(ids, ids_ref), (tok, fam, edges)
            ref = torch.sort(torch.cat([new, d], 1) if cat else new, 1).values
            assert torch.equal(out, ref), (tok, fam, edges, float((out - ref).abs().max()))
            if edges:
                # (the reference's interpolation is discontinuous where a cdf step is below 1e-5, and above the last
                # cdf entry, which the fp32 pdf leaves a few ulp off 1: there a cdf one ulp away - any other
                # implementation's - sends a tie or nextafter(1, 0) to another interval, so the exact checks above
                # are the comparison for these uniforms)
                continue
            for tag, dtype in (("fp32", torch.float32), ("fp64", torch.float64)):
                o = orc.sample_pdf(d.to(dtype), w.to(dtype), u.to(dtype), cat_coarse=cat)
                e = R.nerr64(out, o)
                worst[tag] = max(worst[tag], e)
                assert e < bound, (tok, fam, tag, e, bound)
    _report(f"sample_pdf E={E} n_new={F} {'cat' if cat else 'nocat'} (bound {bound:.1e})", worst)


def test_sample_pdf_edge_cases():
    """n_new = 0 with no uniforms returns the coarse edges; a NaN distance on the last ray of a multi-pass batch sends
    the whole batch to the reference's linspace fallback (and the next clean batch is resampled normally); too much
    shared memory (E = 4097: 262,176 B) and nothing to produce are refused before any launch."""
    L = _L()
    d = R.ray_inputs("translucent", 9, 2)[0].to(DEV)
    w = torch.rand(9, 1, device=DEV)
    out, _, cdf = _sample_pdf(d, w, None, 0, True)
    assert torch.equal(out, d)
    assert bool((cdf[:, 0] == 0).all()) and bool((cdf[:, 1] == 1).all())
    B, E, F = n_rays("P+1"), 65, 129
    d = R.ray_inputs("translucent", B, E)[0]
    w = R.pdf_weights("random", B, E - 1)
    u = torch.rand(B, F, generator=torch.Generator().manual_seed(3))
    dn = d.clone()
    dn[B - 1, 10] = float("nan")
    status = torch.zeros(2, dtype=torch.int32, device=DEV)
    out, _, _ = _sample_pdf(dn.to(DEV), w.to(DEV), u.to(DEV), F, True, status)
    lin = torch.linspace(float(dn[0, 0]), float(dn[0, -1]), E + F).expand(B, -1)
    assert nerr(out.cpu().numpy(), lin.numpy()) < 1e-6
    assert int(status[0]) & 2
    out, _, _ = _sample_pdf(d.to(DEV), w.to(DEV), u.to(DEV), F, True, status)
    assert R.nerr64(out, orc.sample_pdf(d, w.clone(), u)) < R.tol("sample_pdf", E)
    for E, F, cat, code in ((4097, 1, True, E_UNSUPPORTED), (33, 0, False, E_INVALID)):
        d = R.ray_inputs("translucent", 1, E)[0].to(DEV)
        w, u = torch.rand(1, E - 1, device=DEV), torch.rand(1, max(F, 1), device=DEV)
        out = _nan(1, (E if cat else 0) + max(F, 1))
        _refused(code, "neddf_sample_pdf", L.ptr(d), L.ptr(w), L.ptr(u), 1, E, F, 1 if cat else 0, L.ptr(out), None,
                 None, None)
        assert bool(torch.isnan(out).all())


@pytest.mark.parametrize("E,F,cat", PDF_SHAPES)
def test_invert_cdf(E, F, cat):
    """neddf_invert_cdf on the fp32 oracle's cdf: ids and samples bit for bit those of the oracle."""
    L = _L()
    for tok in (["1", "9", "P+1"] if E <= 1025 else ["7"]):
        B = n_rays(tok)
        d = R.ray_inputs("translucent", B, E)[0]
        cdf = orc.pdf_cdf(R.pdf_weights("random", B, E - 1), smooth=not cat)
        u = _uniforms(B, F, E + 1, cdf)
        new_ref, ids_ref = orc.invert_cdf(d, cdf, u)
        dd, cd, ud = d.to(DEV), cdf.to(DEV), u.to(DEV)
        smp, ids = _nan(B, F), torch.full((B, F), -1, dtype=torch.int64, device=DEV)
        _call("neddf_invert_cdf", L.ptr(dd), L.ptr(cd), L.ptr(ud), B, E, F, L.ptr(smp), L.ptr(ids))
        assert torch.equal(ids.cpu(), ids_ref), tok
        assert torch.equal(smp.cpu(), new_ref), tok


# -------------------------------------------------------------------------------------------------- geometry --

def test_coarse_dists_shapes():
    """Stratified edges at the smallest edge counts and at ray counts whose B * E is not a multiple of the block."""
    L = _L()
    for E, B in itertools.product((2, 3, 257), (37, 1000)):
        rc = orc.RenderConfig(sample_coarse=E - 1, dist_near=2.0, dist_far=6.0)
        u = torch.rand(B, E, generator=torch.Generator().manual_seed(E * B))
        ud, out = u.to(DEV), _nan(B, E)
        _call("neddf_coarse_dists", L.ptr(ud), B, E, rc.dist_near, rc.dist_far, L.ptr(out))
        assert nerr(out.cpu().numpy(), orc.coarse_dists(rc, u).numpy()) < 2e-7, (E, B)
        assert nerr(out.cpu().numpy(), orc.coarse_dists(rc, u.double()).numpy()) < 3e-7, (E, B)


def test_make_samples_smallest_edge_counts():
    """Point sampling with one edge per ray; cone sampling with two edges (the far edge of the last one extrapolated,
    ray.py:160-163) and refused with one."""
    L = _L()
    B = 37
    g = torch.Generator().manual_seed(4)
    rd = torch.nn.functional.normalize(torch.randn(B, 3, generator=g), dim=1)
    ro = torch.randn(B, 3, generator=g)
    rdd, rod = rd.to(DEV), ro.to(DEV)
    for kind, E in (("point", 1), ("cone", 2)):
        d = torch.sort(torch.rand(B, E, generator=g) * 4 + 2, 1).values
        dd = d.to(DEV)
        pos, dr, var = _nan(B, E, 3), _nan(B, E, 3), _nan(B, E, 3)
        _call("neddf_make_samples", L.ptr(rdd), L.ptr(rod), L.ptr(dd), B, E, L.SAMPLING_IDS[kind],
              orc.CONE_RAY_RADIUS if kind == "cone" else 0.0, L.ptr(pos), L.ptr(dr), L.ptr(var))
        p_ref, d_ref, v_ref = orc.make_samples(orc.RenderConfig(sampling_type=kind), rd, ro, d)
        p64, _, v64 = orc.make_samples(orc.RenderConfig(sampling_type=kind), rd.double(), ro.double(), d.double())
        assert nerr(pos.cpu().numpy(), p_ref.numpy()) < 1e-6 and nerr(pos.cpu().numpy(), p64.numpy()) < 1e-6, kind
        assert torch.equal(dr.cpu(), d_ref.contiguous()), kind
        if kind == "point":
            assert float(var.abs().max()) == 0.0
        else:
            assert nerr(var.cpu().numpy(), v_ref.numpy()) < 1e-5 and nerr(var.cpu().numpy(), v64.numpy()) < 1e-5
    d = torch.rand(B, 1, device=DEV) + 2
    _refused(E_INVALID, "neddf_make_samples", L.ptr(rdd), L.ptr(rod), L.ptr(d), B, 1, L.SAMPLING_IDS["cone"],
             orc.CONE_RAY_RADIUS, L.ptr(pos), L.ptr(dr), L.ptr(var))


def test_make_image_rays_ranges():
    """A pixel range that starts inside the image and ends exactly at its last pixel, on an image whose sides are
    not multiples of the downsampling; one pixel more is refused."""
    L = _L()
    c = Case("bunny")
    width, height, ds = 803, 611, 7
    w, h = width // ds, height // ds
    first = 1234
    n = w * h - first
    hR, hT = L.fbuf(c.z["cam_R"].reshape(-1)), L.fbuf(c.z["cam_T"].reshape(-1))
    hC = L.fbuf(c.z["cam_calib"].reshape(-1)[:4])
    rd, ro = _nan(n + 1, 3), _nan(n + 1, 3)
    _call("neddf_make_image_rays", width, height, ds, first, n, hR, hT, hC, L.ptr(rd), L.ptr(ro))
    d_ref, o_ref = orc.make_rays(orc.image_uv(width, height, ds)[first:], c.cam)
    assert nerr(rd[:n].cpu().numpy(), d_ref.numpy()) < 1e-6
    assert torch.equal(ro[:n].cpu(), o_ref.contiguous())
    assert bool(torch.isnan(rd[n:]).all())
    _refused(E_INVALID, "neddf_make_image_rays", width, height, ds, first, n + 1, hR, hT, hC, L.ptr(rd), L.ptr(ro))


# -------------------------------------------------------------------------------------------- ray termination --

@pytest.mark.parametrize("tok", ["1", "33", "Q+33"])
def test_terminate_rays_segments(tok):
    """neddf_terminate_rays over segment layouts that split the 40 edges unevenly and end on the closing edge: the
    running transmittance is the product of the compositing factors of each segment, the kept rays are exactly those
    above eps, the executed-evaluation counter counts each live ray's segment.  Q = 1024 rays per SM is one pass."""
    L = _L()
    B, E = n_rays(tok), 40
    g = torch.Generator().manual_seed(B)
    dists = torch.sort(torch.rand(B, E, generator=g) * 4 + 2, dim=1).values
    dens = torch.rand(B, E, generator=g) * 0.3
    dens[::3, 10:14] = 80.0
    fac = (1 - (1 - torch.exp(-dens[:, :-1].double() * (dists[:, 1:] - dists[:, :-1]).double())) + 1e-7)
    dd, sd = dists.to(DEV), dens.to(DEV)
    eps = 1e-2
    for layout in (((0, 12), (12, 12), (24, 16)), ((0, 1), (1, 31), (32, 7), (39, 1)), tuple((j, 1) for j in range(E))):
        trans = torch.ones(B, device=DEV)
        idx = [torch.full((B,), -1, dtype=torch.int32, device=DEV) for _ in range(2)]
        cnt = [torch.zeros(1, dtype=torch.int32, device=DEV) for _ in range(2)]
        ex = torch.zeros(1, dtype=torch.int64, device=DEV)
        cur_i, cur_n, live, expect_ex = None, None, torch.ones(B, dtype=torch.bool), 0
        T = torch.ones(B, dtype=torch.float64)
        for k, (e0, seg) in enumerate(layout):
            _call("neddf_terminate_rays", L.ptr(dd), L.ptr(sd), B, E, e0, seg, L.ptr(cur_i), L.ptr(cur_n), L.ptr(trans),
                  eps, L.ptr(idx[k % 2]), L.ptr(cnt[k % 2]), L.ptr(ex))
            expect_ex += int(live.sum()) * seg
            T = torch.where(live, T * fac[:, e0:min(e0 + seg, E - 1)].prod(1), T)
            live = live & (T > eps)
            n = int(cnt[k % 2].item())
            kept = torch.sort(idx[k % 2][:n].cpu().long()).values
            assert torch.equal(kept, torch.nonzero(live).flatten()), (layout[:3], k)
            # absolute: behind a wall 1 - o is a cancellation in fp32, and T a probability
            assert float((trans.cpu().double() - T).abs().max()) < 1e-5, (layout[:3], k)
            cur_i, cur_n = idx[k % 2], cnt[k % 2]
        assert int(ex.item()) == expect_ex


@pytest.mark.parametrize("engine", ["fp32", "tc", "tc2"])
def test_termination_segments_are_invisible_when_no_ray_stops(engine):
    """An image render with termination on, but eps at half the smallest final transmittance so that no ray can stop,
    is bitwise the render with termination off for 2, 3, 5 and E segments, and executes every nominal evaluation:
    the segment boundaries and the closing edge lose and repeat nothing."""
    import os

    import tests.gpu_util as G
    from tests.helpers import GOLDEN
    z = np.load(os.path.join(GOLDEN, "case_image.npz"))
    c = Case("bunny")
    render, cam = G.build_render(c, engine), G.build_camera(c)
    w, h, ds = int(z["width"]), int(z["height"]), int(z["downsampling"])
    n_pix = (w // ds) * (h // ds)
    g = torch.Generator().manual_seed(int(z["rand_seed"]))
    u = (torch.rand(n_pix, 65, generator=g).to(DEV), torch.rand(n_pix, 129, generator=g).to(DEV))
    keys = ["color", "depth", "transmittance"]
    base = render.render_image(w, h, cam, keys, ds, uniforms=u)
    t_min = float(base["transmittance"].min())
    assert t_min > 0.0
    E = render.sample_coarse + render.sample_fine + 2
    for segments in (2, 3, 5, E):
        render.transmittance_eps, render.termination_segments = 0.5 * t_min, segments
        out = render.render_image(w, h, cam, keys, ds, uniforms=u)
        st = render.termination_stats()
        assert st["executed"] == st["nominal"] == n_pix * E, (segments, st)
        for k in keys:
            assert torch.equal(out[k], base[k]), (segments, k, float((out[k] - base[k]).abs().max()))
    render.check_status()


# ---------------------------------------------------------------------------------------------- end to end --

def _render(c: Case, sc: int, sf: int):
    import neddf_b200
    cfg = {k: v for k, v in c.render_cfg.items() if k != "_target_"}
    cfg.update(sample_coarse=sc, sample_fine=sf)
    r = neddf_b200.NeRFRender(network_config=c.net_cfg, **cfg)
    r.load_state_dict(c.state_dict())
    r.to(DEV)
    r.set_iter(c.iter)
    r.set_engine("fp32")
    return r, orc.RenderConfig(**cfg)


@pytest.mark.parametrize("sc,sf", [(1, 0), (31, 33), (64, 128), (384, 384), (1024, 1024)])
def test_render_rays_sample_counts(sc, sf):
    """render_rays at other sample counts than the golden cases': the no-grad forward against the fp32 oracle, and the
    parameter gradients of a training step against fp32 autograd through the same oracle.  At (384, 384) the
    compositing backward's shared memory is above 48 KB, at (1024, 1024) that of the resampling too."""
    import tests.gpu_util as G
    c = Case("bunny")
    render, rc = _render(c, sc, sf)
    cam = G.build_camera(c)
    Ef = sc + sf + 2
    g = torch.Generator().manual_seed(sc * 7 + sf)
    n = 24 if Ef < 500 else 4
    uv = c.t("uv")[:n]
    u_c, u_f = torch.rand(n, sc + 1, generator=g), torch.rand(n, sf + 1, generator=g)
    with torch.no_grad():
        out = render.render_rays(uv.to(DEV), cam, uniforms=(u_c.to(DEV), u_f.to(DEV)))
        ref = orc.render_rays(c.p_coarse, c.p_fine, c.fc, c.st, rc, uv, c.cam, u_c, u_f)
        ref64 = orc.render_rays(c.p_coarse, c.p_fine, c.fc, c.st, rc, uv, c.cam, u_c, u_f, dtype=torch.float64)
    errs = {}
    for k, v in ref.items():
        tol = 1e-3 if k == "weight" else PARITY_TOL
        # from about 800 samples per ray the fp32 oracle itself moves away from exact arithmetic by more than the
        # parity bound (fields_penalty 2.3e-4 at (384, 384), weight 1e-3 at (1024, 1024)): there the bound is
        # twice the oracle's own distance, against the fp64 run
        tol = max(tol, 2 * nerr(v.numpy(), ref64[k].numpy()))
        errs[k] = nerr(out[k].cpu().numpy(), ref64[k].numpy())
        assert_parity(out[k].cpu().numpy(), ref64[k].numpy(), tol, c.kinked, k)
        assert_parity(out[k].cpu().numpy(), v.numpy(), tol, c.kinked, k)
    _report(f"render_rays ({sc}, {sf}) forward against fp64", errs)
    n = 4
    P = {k: v.clone().requires_grad_(True) for k, v in c.p_fine.items()}
    assert not c.separate
    ref = orc.render_rays(P, P, c.fc, c.st, rc, uv[:n], c.cam, u_c[:n], u_f[:n])
    loss_of = lambda o: (o["color"].sum() + 0.1 * o["depth"].sum() + 0.05 * o["transmittance"].sum()  # noqa: E731
                         + 0.01 * o["fields_penalty"].sum() + 0.1 * o["color_coarse"].sum())
    loss_of(ref).backward()
    render.zero_grad()
    out = render.render_rays(uv[:n].to(DEV), cam, uniforms=(u_c[:n].to(DEV), u_f[:n].to(DEV)))
    loss_of(out).backward()
    errs = {}
    for name, p in render.network_fine.named_parameters():
        errs[name] = nerr(p.grad.cpu().numpy(), P[name].grad.numpy())
    # as test_render_rays_training_matches_reference_gradients
    assert max(errs.values()) < 2e-4, {k: v for k, v in errs.items() if v >= 2e-4}
    _report(f"render_rays ({sc}, {sf}) gradients, worst", {"grad": max(errs.values())})


def test_render_rays_beyond_the_training_backward():
    """At (2048, 2048) samples the forward runs; a training render is refused before it starts, since the
    compositing backward of its 4098 fine edges would need more than 200 KB of shared memory."""
    import tests.gpu_util as G
    from neddf_b200 import render as render_mod
    assert render_mod.COMPOSITE_BACKWARD_MAX_EDGES == 3201  # the largest E of test_composite_backward; 3202 is refused
    c = Case("bunny")
    render, rc = _render(c, 2048, 2048)
    cam = G.build_camera(c)
    n = 2
    g = torch.Generator().manual_seed(2048)
    uv, u_c, u_f = c.t("uv")[:n], torch.rand(n, 2049, generator=g), torch.rand(n, 2049, generator=g)
    with torch.no_grad():
        out = render.render_rays(uv.to(DEV), cam, uniforms=(u_c.to(DEV), u_f.to(DEV)))
    ref = orc.render_rays(c.p_coarse, c.p_fine, c.fc, c.st, rc, uv, c.cam, u_c, u_f)
    for k in ("color", "depth", "transmittance", "color_coarse"):
        assert nerr(out[k].cpu().numpy(), ref[k].numpy()) < PARITY_TOL, k
    with pytest.raises(RuntimeError, match="training backward"):
        render.render_rays(uv.to(DEV), cam, uniforms=(u_c.to(DEV), u_f.to(DEV)))


# --------------------------------------------------------------------------------- image chunking and shards --

@pytest.mark.parametrize("engine", ["fp32", "tc"])
def test_render_pixels_chunks_and_shards(engine):
    """render_image is bitwise the same for any launch size (image_chunk), and the pixel shards of dist.shard_range
    for two and three ranks concatenate to the full image bit for bit, which the multi-GPU render relies on."""
    import os

    import tests.gpu_util as G
    from neddf_b200 import dist
    from tests.helpers import GOLDEN
    z = np.load(os.path.join(GOLDEN, "case_image.npz"))
    c = Case("bunny")
    render, cam = G.build_render(c, engine), G.build_camera(c)
    w, h, ds = int(z["width"]), int(z["height"]), int(z["downsampling"])
    n_pix = (w // ds) * (h // ds)
    g = torch.Generator().manual_seed(5)
    u = (torch.rand(n_pix, 65, generator=g).to(DEV), torch.rand(n_pix, 129, generator=g).to(DEV))
    keys = ["color", "depth", "transmittance", "color_coarse"]
    base = render.render_image(w, h, cam, keys, ds, uniforms=u)
    for chunk in (37, 4096):
        render.image_chunk = chunk
        out = render.render_image(w, h, cam, keys, ds, uniforms=u)
        for k in keys:
            assert torch.equal(out[k], base[k]), (chunk, k)
    render.image_chunk = 163840
    render.network_coarse.eval()
    render.network_fine.eval()
    for world in (2, 3):
        parts = []
        for rank in range(world):
            first, count = dist.shard_range(n_pix, world, rank)
            parts.append(render.render_pixels(w, h, cam, keys, ds, first, count,
                                              uniforms=(u[0][first:first + count], u[1][first:first + count])))
        for k in keys:
            full = torch.cat([p[k] for p in parts], 0).reshape(base[k].shape)
            assert torch.equal(full, base[k]), (world, k)
    render.check_status()


# ---------------------------------------------------------------------------------------------- training loss --

@pytest.mark.parametrize("B", [1, 31, 256, 257, 100003])
def test_render_loss(B):
    """neddf_render_loss: the six terms and the gradients of their sum against fp64 autograd through the reference's
    objective, with every weight on and with each weight zero in turn (its term and its gradient exactly 0)."""
    L = _L()
    import bench
    g = torch.Generator().manual_seed(B)
    names = ("color", "color_coarse", "transmittance", "transmittance_coarse", "fields_penalty",
             "fields_penalty_coarse")
    out = {k: torch.rand(B, 3, generator=g) if k.startswith("color") else torch.rand(B, generator=g) for k in names}
    out["transmittance"][:5] = torch.tensor([0.0, 1.0, 1e-8, 1 - 1e-8, 0.5])[:B]  # both sides of the clamp
    tc, tm = torch.rand(B, 3, generator=g), (torch.rand(B, generator=g) > 0.4).float()
    w_full = [bench.LOSS_W["color"][0], bench.LOSS_W["color"][1], bench.LOSS_W["mask"][0], bench.LOSS_W["mask"][1],
              bench.LOSS_W["fields_penalty"][0], bench.LOSS_W["fields_penalty"][1]]
    with torch.no_grad():  # the term-by-term restatement sums to bench.train_loss
        total = float(sum(R.loss_terms(out, tc, tm, w_full, torch.float32)))
        assert abs(total - float(bench.train_loss(out, tc, tm))) < 1e-6 * abs(total)
    dv = {k: v.to(DEV) for k, v in out.items()}
    tcd, tmd = tc.to(DEV), tm.to(DEV)
    worst = 0.0
    for zero in (None, 0, 1, 2, 3, 4, 5):
        w = list(w_full)
        if zero is not None:
            w[zero] = 0.0
        wd = torch.tensor(w, device=DEV)
        terms = torch.full((6,), float("nan"), device=DEV)
        grads = {k: torch.full_like(v, float("nan")) for k, v in dv.items()}
        _call("neddf_render_loss", *[L.ptr(dv[k]) for k in names], L.ptr(tcd), L.ptr(tmd), B, L.ptr(wd), L.ptr(terms),
              *[L.ptr(grads[k]) for k in names])
        o64 = {k: v.double().requires_grad_(True) for k, v in out.items()}
        ref = R.loss_terms(o64, tc, tm, w, torch.float64)
        sum(ref).backward()
        for k in range(6):
            r, t = float(ref[k]), float(terms[k])
            assert abs(t - r) <= R.LOSS_TOL * abs(r), (zero, k, t, r)
            if k == zero:
                assert t == 0.0
        for i, k in enumerate(names):
            e = R.nerr64(grads[k], o64[k].grad)
            worst = max(worst, e)
            assert e < R.LOSS_TOL, (zero, k, e)
            if zero is not None and names.index(k) == zero:
                assert bool((grads[k] == 0).all()), (zero, k)
    _report(f"render_loss B={B}", {"grad": worst})
