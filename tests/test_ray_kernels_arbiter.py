"""fp64 arbiter for the bounds of tests/test_ray_kernels_gpu.py: every input family of tests/ray_cases.py through the
fp32 oracle and the fp64 oracle on the CPU.  The GPU tests hold the kernels to tests.ray_cases.tol(kind, E) against
both; this file shows that the reference's own fp32 arithmetic needs that much on the same inputs, and no more than
about half of it, so a kernel that passes is as close to exact arithmetic as the computation it restates."""
import pytest
import torch

from oracle import neddf_oracle as orc
from tests import ray_cases as R

# (E, B): edge counts the GPU file composites, at ray counts large enough for the worst ray to show
COMPOSITE_SHAPES = [(2, 1024), (3, 1024), (33, 1024), (194, 1024), (770, 128), (1537, 32), (3201, 16)]
PDF_SHAPES = [(2, 1, True), (2, 1, False), (3, 1, False), (33, 33, True), (33, 31, False), (65, 129, True),
              (65, 448, True), (65, 513, False), (1025, 1025, True), (2049, 2049, True)]


@pytest.mark.parametrize("family", R.FAMILIES)
def test_composite_fp32_against_fp64(family):
    worst = []
    for E, B in COMPOSITE_SHAPES:
        d, s, c, p = R.ray_inputs(family, B, E)
        a = R.composite_ref(d, s, c, p, torch.float32)
        b = R.composite_ref(d, s, c, p, torch.float64)
        e = max(R.nerr64(a[k], b[k]) for k in a)
        g = R.upstream(B, E)
        ga = R.composite_grad_ref(d, s, c, p, g, torch.float32)
        gb = R.composite_grad_ref(d, s, c, p, g, torch.float64)
        eg = max(R.nerr64(x, y) for x, y in zip(ga, gb))
        worst.append((E, e, eg))
        assert e < 0.5 * R.tol("composite", E), (family, E, e)
        assert eg < 0.5 * R.tol("composite_grad", E), (family, E, eg)
    print(f"[arbiter] composite {family}: " + ", ".join(f"E={E} {e:.1e} / grad {eg:.1e}" for E, e, eg in worst))


@pytest.mark.parametrize("family", R.PDF_FAMILIES)
def test_sample_pdf_fp32_against_fp64(family):
    worst = []
    for E, F, cat in PDF_SHAPES:
        B = 4096 if E < 1000 else (1024 if E < 2000 else 16)  # the worst of thousands of rays, as on the GPU
        d = R.ray_inputs("translucent", B, E)[0]
        w = R.pdf_weights(family, B, E - 1)
        u = torch.rand(B, F, generator=torch.Generator().manual_seed(E + F))
        a = orc.sample_pdf(d, w.clone(), u, cat_coarse=cat)
        b = orc.sample_pdf(d.double(), w.double(), u.double(), cat_coarse=cat)
        e = R.nerr64(a, b)
        worst.append((E, F, cat, e))
        assert e < 0.5 * R.tol("sample_pdf", E), (family, E, F, cat, e)
    print(f"[arbiter] sample_pdf {family}: " + ", ".join(f"({E},{F},{'cat' if c else 'nocat'}) {e:.1e}"
                                                       for E, F, c, e in worst))


def test_loss_fp32_against_fp64():
    g = torch.Generator().manual_seed(5)
    for B in (1, 257, 100003):
        out = {k: torch.rand(B, 3, generator=g) if k.startswith("color") else torch.rand(B, generator=g)
               for k in ("color", "color_coarse", "transmittance", "transmittance_coarse", "fields_penalty",
                         "fields_penalty_coarse")}
        out["transmittance"][:5] = torch.tensor([0.0, 1.0, 1e-8, 1 - 1e-8, 0.5])[:B]  # both sides of the clamp
        tc, tm = torch.rand(B, 3, generator=g), (torch.rand(B, generator=g) > 0.4).float()
        w = [1.0, 0.1, 0.05, 0.005, 0.01, 0.01]
        o32 = {k: v.clone().requires_grad_(True) for k, v in out.items()}
        o64 = {k: v.double().requires_grad_(True) for k, v in out.items()}
        a = R.loss_terms(o32, tc, tm, w, torch.float32)
        b = R.loss_terms(o64, tc, tm, w, torch.float64)
        for k in range(6):
            assert abs(float(a[k]) - float(b[k])) <= 0.5 * R.LOSS_TOL * abs(float(b[k])), (B, k)
        sum(a).backward()
        sum(b).backward()
        for k in out:
            assert R.nerr64(o32[k].grad, o64[k].grad) < 0.5 * R.LOSS_TOL, (B, k)
