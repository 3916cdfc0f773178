"""Inputs and tolerances of the ray kernels on either side of the field network: compositing and its backward,
hierarchical resampling, coarse edges and sample geometry, the training objective.

Shared by tests/test_ray_kernels_gpu.py (the CUDA kernels against the oracle in fp32 and in fp64) and
tests/test_ray_kernels_arbiter.py, which runs every input family through the fp32 oracle and the fp64 oracle on the CPU
and asserts that they agree within the same bounds: each tolerance below is what the reference's own fp32 arithmetic
needs on these inputs, not a number picked to make a kernel pass."""
import numpy as np
import torch

from oracle import neddf_oracle as orc

MAX_DIST = 6.0

# max|new - ref| / max|ref| (tests.helpers.nerr) per output, as (floor, per edge): the bound at E edges per ray is
# max(floor, per_edge * E).  The reference's fp32 arithmetic rounds every factor of the transmittance product and every
# entry of the cdf, so its distance from exact arithmetic grows linearly with the number of edges; the arbiter measures
# it and each pair below is at least twice the largest distance it sees (tests/test_ray_kernels_arbiter.py).
TOL = {
    "composite": (1e-6, 6e-8),       # weight, depth, colour, transmittance, penalty integral
    "composite_grad": (1e-6, 1e-7),  # d density, d colour, d penalty through autograd
    "sample_pdf": (5e-6, 2e-6),      # resampled distances: a cdf error moves a sample by error / pdf of its interval
}


def tol(kind: str, n_edges: int) -> float:
    floor, per_edge = TOL[kind]
    return max(floor, per_edge * n_edges)


# the density families: translucent media, opaque walls that drive each factor 1 - o + 1e-7 to its 1e-7 floor,
# empty space (T = 1, depth = max_dist exactly), saturated densities (o = 1 exactly), and repeated edges (delta = 0,
# which sample_pdf produces whenever a uniform equals a cdf entry)
FAMILIES = ("translucent", "wall", "zero", "huge", "dup")


def ray_inputs(family: str, B: int, E: int, seed: int = 0):
    """(dists [B,E] ascending in [2, 6], density [B,E], color [B,E,3], penalty [B,E]) in fp32."""
    g = torch.Generator().manual_seed(seed * 7919 + E * 31 + B)
    dists = torch.sort(torch.rand(B, E, generator=g) * 4 + 2, dim=1).values
    density = torch.rand(B, E, generator=g) * 0.3
    color = torch.rand(B, E, 3, generator=g)
    penalty = torch.randn(B, E, generator=g)
    if family == "wall":
        # optical depth sigma * delta = 80 on three intervals: exp(-80) vanishes next to 1 in fp32, so o = 1 and the
        # factor sits at its floor of 1e-7 (a wall that left exp(-sigma delta) near 1e-7 would instead make the
        # reference's 1 - o a cancellation, ill-conditioned in any precision below fp64)
        j0 = E // 3
        delta = (dists[:, 1:] - dists[:, :-1])[:, j0:j0 + 3]
        density[:, j0:j0 + delta.shape[1]] = 80.0 / delta.clamp_min(1e-30)
    elif family == "zero":
        density.zero_()
    elif family == "huge":
        density.fill_(1e30)
    elif family == "dup":
        if E >= 3:
            dists[:, 1::3] = dists[:, 0:-1:3][:, :dists[:, 1::3].shape[1]]
            dists = torch.sort(dists, dim=1).values
    elif family != "translucent":
        raise ValueError(family)
    return dists.contiguous(), density.contiguous(), color.contiguous(), penalty.contiguous()


def composite_ref(dists, density, color, penalty, dtype):
    """Every output of neddf_composite from the oracle, with the inputs cast to ``dtype``."""
    d, s, c, p = (t.to(dtype) for t in (dists, density, color, penalty))
    out = orc.composite(d, s, c, MAX_DIST)
    out["fields_penalty"] = orc.integrate_penalty(d, p)
    return out


def upstream(B: int, E: int, seed: int = 1):
    """Random upstream gradients of weight, depth, colour, transmittance and the penalty integral."""
    g = torch.Generator().manual_seed(seed * 104729 + E * 17 + B)
    return {"weight": torch.randn(B, E - 1, generator=g), "depth": torch.randn(B, generator=g),
            "color": torch.randn(B, 3, generator=g), "transmittance": torch.randn(B, generator=g),
            "fields_penalty": torch.randn(B, generator=g)}


def composite_grad_ref(dists, density, color, penalty, g, dtype):
    """(d density, d colour, d penalty) by autograd through the oracle in ``dtype``."""
    s, c, p = (t.detach().to(dtype).clone().requires_grad_(True) for t in (density, color, penalty))
    out = composite_ref(dists, s, c, p, dtype)
    loss = sum((out[k] * g[k].to(dtype)).sum() for k in g)
    loss.backward()
    return s.grad, c.grad, p.grad


# weight families of sample_pdf (the coarse weights are sanitised in place: negative -> -0.0, NaN -> 0)
PDF_FAMILIES = ("random", "zero", "onehot", "negative", "nan", "denormal")


def pdf_weights(family: str, B: int, n_w: int, seed: int = 0):
    g = torch.Generator().manual_seed(seed * 6151 + n_w * 13 + B)
    w = torch.rand(B, n_w, generator=g) ** 3
    if family == "zero":
        w.zero_()
    elif family == "onehot":
        w.zero_()
        w[torch.arange(B), torch.randint(0, n_w, (B,), generator=g)] = 1e30
    elif family == "negative":
        w[:, ::2] = -w[:, ::2]
    elif family == "nan":
        w[:, ::5] = float("nan")
    elif family == "denormal":
        w[:, ::2] = 1e-40
    elif family != "random":
        raise ValueError(family)
    return w.contiguous()


def nerr64(new, ref) -> float:
    """tests.helpers.nerr on tensors, where a tensor whose largest entry is below 1e-25 counts as zero: behind a wall
    of optical depth 80 a gradient is d o / d sigma = delta exp(-80) ~ 1e-35 in autograd, and exactly 0 where 1 - o
    is rounded to fp32 first, as the kernels and the reference's forward do."""
    new = np.asarray(new.detach().cpu(), dtype=np.float64)
    ref = np.asarray(ref.detach().cpu(), dtype=np.float64)
    assert new.shape == ref.shape, (new.shape, ref.shape)
    den = max(float(np.abs(ref).max()) if ref.size else 0.0, 1e-25)
    return float(np.abs(new - ref).max() / den) if ref.size else 0.0


def loss_terms(out, t_color, t_mask, w, dtype):
    """The six weighted terms of the reference's objective (bench.train_loss, term by term) in ``dtype``:
    colour MSE, mask BCE on 1 - T clamped to [1e-6, 1 - 1e-6], mean penalty; fine then coarse.  The clamp bounds are
    those of the reference's fp32 tensors, in any ``dtype``: 1 - 1e-6 is 1 - 1.013e-6 in fp32, and -log(1 - m) at the
    bound differs by 1 % between the two."""
    lo, hi = (float(torch.tensor(v, dtype=torch.float32)) for v in (1e-6, 1.0 - 1e-6))
    terms = []
    for k, suffix in ((0, ""), (1, "_coarse")):
        terms.append(w[k] * torch.mean(torch.square(out["color" + suffix].to(dtype) - t_color.to(dtype))))
    for k, suffix in ((2, ""), (3, "_coarse")):
        m = torch.clamp(1.0 - out["transmittance" + suffix].to(dtype), lo, hi)
        y = t_mask.to(dtype)
        terms.append(w[k] * -torch.mean(y * torch.log(m) + (1.0 - y) * torch.log(1.0 - m)))
    for k, suffix in ((4, ""), (5, "_coarse")):
        terms.append(w[k] * torch.mean(out["fields_penalty" + suffix].to(dtype)))
    return terms


# relative bound of each loss term and of its gradients (one fp32 rounding per element, sums in fp64)
LOSS_TOL = 1e-6
