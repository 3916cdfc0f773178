"""Golden vectors of BaseNeuralRender.sample_pdf from the REAL reference (neddf/render/base_neural_render.py:27-115) at
the smallest edge counts, E = 2 (one interval) and E = 3, in both modes; imported from /root/reference in the build
container with the hydra / omegaconf stand-ins of tests/golden/_refstub, the internal torch.rand replaced by recorded
uniforms.  At one interval the neighbour-max smoothing of cat_coarse=False (:61-68) writes the empty slice
weights[:, 1:-1] and so changes nothing.

    python tests/golden/make_pdf_small_golden.py      ->  tests/golden/case_pdf_small.npz
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "_refstub"))
sys.path.insert(0, "/root/reference")

from neddf.render.base_neural_render import BaseNeuralRender  # noqa: E402


class _R(BaseNeuralRender):  # the abstract bits are not on this path
    def render_rays(self, *a, **k):
        raise NotImplementedError

    def get_parameters_list(self):
        return []

    def render_image(self, *a, **k):
        raise NotImplementedError

    def render_field_slice(self, *a, **k):
        raise NotImplementedError

    def get_network(self):
        return None


g = torch.Generator().manual_seed(12)
B, F = 6, 5
arrays = {}
for E in (2, 3):
    dists = torch.sort(torch.rand(B, E, generator=g) * 4 + 2, dim=1).values
    w = torch.rand(B, E - 1, generator=g) ** 3
    w[1, 0] = -0.2           # sanitised in place (:52-55)
    w[3, E - 2] = float("nan")
    w[4] = 0.0
    u = torch.rand(B, F, generator=g)
    u[5, 0] = 0.0
    arrays[f"e{E}_dists"], arrays[f"e{E}_weights"], arrays[f"e{E}_u"] = dists.numpy(), w.numpy(), u.numpy()
    for cat in (True, False):
        orig = torch.rand
        torch.rand = lambda *s, **k: u.clone()
        try:
            w_in = w.clone()
            out = _R().sample_pdf(dists.clone(), w_in, F, cat_coarse=cat)
        finally:
            torch.rand = orig
        tag = f"e{E}_{'cat' if cat else 'nocat'}"
        arrays[tag + "_out"], arrays[tag + "_weights_after"] = out.numpy(), w_in.numpy()
np.savez(os.path.join(HERE, "case_pdf_small.npz"), **arrays)
print("wrote case_pdf_small.npz", sorted(arrays))
