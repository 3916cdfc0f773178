"""fp64 arbiter for the two parity allowances the GPU tests use (VERDICT round 1, weak items 1 and 3).

The GPU tests hold every tensor to max|new - ref| / max|ref| <= 1e-4 except
  (a) per-sample fine `weight`s end to end (1e-3; stage-wise 1e-4), and
  (b) configurations with piecewise-linear hidden activations (ReLU / LeakyReLU): all but <= 1 % of the elements.
Both allowances are properties of the REFERENCE's arithmetic, not of the CUDA path.  This file shows it on the CPU with
the reference restatement alone: fp32 against its own fp64 run and against itself fed inputs shifted by one ulp."""
import numpy as np
import torch

from oracle import neddf_oracle as orc
from tests.helpers import Case, nerr


def _kink_distance(c: Case, pos, dd, var) -> np.ndarray:
    """Per sample: smallest |pre-activation| over all hidden units (fp64 run)."""
    taps = {}
    P64 = {k: v.double() for k, v in c.p_fine.items()}
    orc.field_forward(P64, c.fc, c.st, pos.double(), dd.double(), var.double(), taps=taps)
    pre = [v.abs().min(1).values for k, v in taps.items() if k.endswith("_pre")]
    return torch.stack(pre).min(0).values.reshape(pos.shape[:2]).numpy()


def test_fine_weights_amplify_coarse_differences():
    """(a) The reference in fp32 against its fp64 run on the pretrained bunny_smoke case: the coarse weights agree to
    ~4e-6, every integrated output to <= 1e-5 - but the per-sample FINE weights only to ~5e-5, because they are
    compared at resampled positions (sample_pdf inverts the coarse cdf, base_neural_render.py:70-100) where the density
    has steep fronts.  A >= 10x amplification of coarse-pass differences: a path whose coarse weights differ from the
    reference's by 1e-5 (any reordered fp32 sum does) cannot promise 1e-4 on that tensor; 1e-3 is the honest bound."""
    c = Case("bunny")
    args = (c.p_coarse, c.p_fine, c.fc, c.st, c.rc, c.t("uv"), c.cam, c.t("u_coarse"), c.t("u_fine"))
    with torch.no_grad():
        a = orc.render_rays(*args)
        r = orc.render_rays(*args, dtype=torch.float64)
    e = {k: nerr(a[k].numpy(), r[k].numpy()) for k in a}
    assert e["weight_coarse"] < 1e-5
    for k in ("color", "depth", "transmittance", "color_coarse", "depth_coarse", "transmittance_coarse"):
        assert e[k] < 1e-5, (k, e[k])
    assert e["weight"] > 5 * e["weight_coarse"], e  # measured 5.5e-5 vs 4.3e-6
    assert 2e-5 < e["weight"] < 1e-3, e  # the reference's own fp32 already uses half of a 1e-4 budget


def test_kinked_outliers_sit_on_kinks():
    """(b) LeakyReLU golden configuration, the reference restatement in fp32 at the golden positions and at positions
    shifted by ONE ulp: distance / density / colour agree to 1e-4, but `fields_penalty` (built from Jacobian rows,
    neddf.py:259-300) jumps by up to 3e-4 on a few samples - and every one of them has a hidden pre-activation within
    the shift's reach of zero in the fp64 run (the slope of that unit flips).  The smooth tanhExp network shows none.
    The GPU tests' allowance for kinked configurations (<= 1 % of the elements, capped at 5e-2) covers exactly this."""
    outliers = {}
    for name in ("leaky", "point", "bunny"):
        c = Case(name)
        d, o = orc.make_rays(c.t("uv"), c.cam)
        pos, dd, var = orc.make_samples(c.rc, d, o, c.t("dists_fine"))
        pos2 = torch.nextafter(pos, torch.full_like(pos, float("inf")))
        with torch.no_grad():
            a = orc.field_forward(c.p_fine, c.fc, c.st, pos, dd, var)
            b = orc.field_forward(c.p_fine, c.fc, c.st, pos2, dd, var)
        kink = _kink_distance(c, pos, dd, var)
        n_bad = 0
        for k in ("distance", "density", "color", "fields_penalty", "aux_grad"):
            err = ((a[k] - b[k]).abs() / a[k].abs().max()).numpy()
            if err.ndim == 3:
                err = err.max(-1)
            bad = np.argwhere(err >= 1e-4)
            n_bad += len(bad)
            assert len(bad) <= max(2, err.size // 100) and float(err.max()) < 5e-2, (name, k)
            # one ulp of position is amplified by the positional encoding (2^9) into a pre-activation shift of <= 1e-4
            assert all(kink[tuple(i)] < 1e-4 for i in bad), (name, k, [(tuple(i), kink[tuple(i)]) for i in bad])
            if k in ("distance", "density", "aux_grad"):
                assert len(bad) == 0, (name, k)
        outliers[name] = n_bad
    assert outliers["bunny"] == 0, outliers  # smooth activation: no exemption needed, none granted (Case.kinked is False)
    assert outliers["leaky"] > 0, outliers   # measured: 3 of 1552 samples, kink distances <= 2.4e-6


def test_reference_gradients_against_the_fp64_arbiter():
    """Gradient parity budget (VERDICT round 1, weak 1).  The gradients the REAL reference's hand-written backward
    produced in fp32 (golden case_train, 26 tensors, loss over both passes) against the oracle's fp64 autograd run of
    the same step: the reference itself sits at ~2.4e-6 of the exact gradients, the fp32 restatement at the same
    distance and at 6e-7 of the reference.  The CUDA training path is measured at 1.6e-6 .. 3.5e-5 of fp64
    (tools/grad_err.py) - inside the 1e-4 the GPU tests assert
    (test_field_backward_matches_autograd; 2e-4 end to end through the resampling)."""
    c = Case("train")

    def grads(dtype):
        p = {k: v.clone().to(dtype).requires_grad_(True) for k, v in c.p_fine.items()}
        out = orc.render_rays(p, p, c.fc, c.st, c.rc, c.t("uv"), c.cam, c.t("u_coarse"), c.t("u_fine"), dtype=dtype)
        loss = (out["color"].sum() + 0.1 * out["depth"].sum() + 0.05 * out["transmittance"].sum()
                + 0.01 * out["fields_penalty"].sum() + 0.1 * out["color_coarse"].sum()
                + 0.001 * out["fields_penalty_coarse"].sum())  # the loss of tests/golden/make_golden.py
        loss.backward()
        return {k: v.grad.numpy() for k, v in p.items()}

    g64, g32 = grads(torch.float64), grads(torch.float32)
    worst_ref, worst_32 = 0.0, 0.0
    for k, exact in g64.items():
        ref = c.z["grad_network_fine." + k]
        a, b = exact, g32[k]
        if a.ndim == 2 and a.shape[1] > 3:  # the fixture keeps every 8th input row of the big matrices
            a, b = a[::8], b[::8]
        worst_ref = max(worst_ref, nerr(ref, a))
        worst_32 = max(worst_32, nerr(b, a))
    assert worst_ref < 2e-5 and worst_32 < 2e-5, (worst_ref, worst_32)  # measured 2.4e-6 / 2.5e-6
    assert worst_ref > 1e-7  # and not zero: fp32 has a floor, the 1e-4 bar leaves it a factor ~40
