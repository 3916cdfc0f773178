#!/usr/bin/env python
"""Golden fixtures for NeDDF at structures other than the default one, from the REAL reference.

Run in the build container only (needs /root/reference):

    python tests/golden/make_field_config_golden.py

For configurations of tests/field_configs.py it builds the reference's own NeDDF (neddf/network/neddf.py) with that
configuration, loads the seeded parameters of ``field_configs.params`` (the file keeps the seed, not the weights),
applies ``set_iter`` and runs ``forward`` on fixed Sampling tensors with autograd.  The loss is
sum(density * g_density) + sum(color * g_color) + sum(fields_penalty * g_penalty) for recorded random upstream
gradients, differentiated by the reference's hand-written autograd Functions.  Stored in case_cfg_<name>.npz: the
configuration, seed and iteration, the inputs, the upstream gradients, the five outputs and the parameter gradients
(of the 256-wide matrices every 8th input row and 4th output column, ``fixture_sample``).
  C2_minimal   ranks 1 / 1, one hidden layer per trunk, no skip, LeakyReLU hidden, tanhExp density
  C7_deepest   ranks 6 / 2, 12 + 12 hidden layers, skips [0, 5, 10], LeakyReLU hidden and density
"""
import importlib.util
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402,F401  (sets sys.path for the reference + stubs)

import numpy as np  # noqa: E402
import torch  # noqa: E402
# tests/field_configs.py by path: on this sys.path `tests` is the reference's own test package
_spec = importlib.util.spec_from_file_location("field_configs", os.path.join(os.path.dirname(HERE), "field_configs.py"))
fcfg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(fcfg)
from neddf.network import NeDDF  # noqa: E402  (reference)
from neddf.ray import Sampling  # noqa: E402  (reference)

NAMES = ["C2_minimal", "C7_deepest"]
B, S = 2, 24


def fixture_sample(g):
    """The stored part of a parameter gradient (the test applies the same selection)."""
    return g[::8, ::4] if (g.ndim == 2 and g.shape[1] > 3) else g


def record(name):
    kw = fcfg.kwargs(name)
    net = NeDDF(**kw)
    print(name, "load:", net.load_state_dict(fcfg.params(name)))
    it = fcfg.CONFIGS[name]["iter"]
    net.set_iter(it)
    pos, dirs, var = fcfg.samples(B, S, fcfg.SEED[name] + 1)
    gd, gc, gp = fcfg.upstream(B, S, fcfg.SEED[name] + 2)
    out = net(Sampling(pos.clone(), dirs.clone(), var.clone()))
    loss = (out["density"] * gd).sum() + (out["color"] * gc).sum() + (out["fields_penalty"] * gp).sum()
    net.zero_grad()
    loss.backward()
    res = dict(cfg=np.array(json.dumps(dict(name=name, kw=kw, iter=it, seed=fcfg.SEED[name]))),
               pos=pos.numpy(), dirs=dirs.numpy(), var=var.numpy(), g_density=gd.numpy(), g_color=gc.numpy(),
               g_penalty=gp.numpy())
    for k, v in out.items():
        res["out_" + k] = v.detach().numpy()
    for k, p in net.named_parameters():
        res["grad_" + k] = fixture_sample(p.grad.detach().numpy())
    np.savez_compressed(os.path.join(HERE, f"case_cfg_{name}.npz"), **res)
    print(name, "done", {k: float(np.abs(v).max()) for k, v in res.items() if k.startswith("out_")})


if __name__ == "__main__":
    torch.set_num_threads(8)
    for n in NAMES:
        record(n)
