"""CPU: the network structures of tests/field_configs.py on the host side - the C ABI's layer table and its
rejections, the hand-derived backward (tests/manual_backward.py, the CPU twin of field_bwd.cu) against fp64 autograd
through the oracle, and the oracle against the real reference at a minimal and at the deepest structure."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import neddf_oracle as orc
from tests import field_configs as fcfg
from tests.helpers import GOLDEN, assert_parity, nerr
from tests.manual_backward import field_backward

NEDDF_E_INVALID, NEDDF_E_UNSUPPORTED = -1, -3


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from neddf_b200 import _lib as L
    return L.lib()


def _shapes(lib, net):
    cfg = net._config_struct()
    buf = (C.c_int32 * 128)()
    n = lib.neddf_field_layer_shapes(C.byref(cfg), buf, 64)
    return n, [(buf[2 * i], buf[2 * i + 1]) for i in range(max(n, 0))]


@pytest.mark.parametrize("name", fcfg.NAMES)
def test_layer_table_matches_oracle_and_module(lib, name):
    import neddf_b200
    net = neddf_b200.NeDDF(**fcfg.kwargs(name))
    n, got = _shapes(lib, net)
    ref = orc.layer_shapes(fcfg.field_config(name))
    assert n == len(ref) == (net.ddf_layer_count - 1) + (net.col_layer_count - 1) + 3
    assert got == [(a, b) for _, a, b in ref]
    sd = net.state_dict()
    assert set(sd) == {f"{k}.{p}" for k, _, _ in ref for p in ("weight", "bias")}
    for k, a, b in ref:
        assert tuple(sd[k + ".weight"].shape) == (a, b) and tuple(sd[k + ".bias"].shape) == (b,), k
    net.load_state_dict(fcfg.params(name))  # strict: the seeded parameters fit the module exactly


def test_structure_limits_are_refused_before_any_launch(lib):
    """The limits are enforced by the configuration check that both neddf_field_layer_shapes and neddf_field_create
    run first (no CUDA call is made for a refused configuration)."""
    import neddf_b200

    def codes(**kw):
        cfg = neddf_b200.NeDDF(**kw)._config_struct()
        h = C.c_void_p()
        rc_create = lib.neddf_field_create(C.byref(cfg), C.byref(h))
        assert not h.value
        return lib.neddf_field_layer_shapes(C.byref(cfg), None, 0), rc_create

    # 12 + 13 = 25 hidden layers, one more than a field describes
    assert codes(embed_pos_rank=6, embed_dir_rank=2, ddf_layer_count=13, col_layer_count=14, skips=[]) == \
        (NEDDF_E_UNSUPPORTED, NEDDF_E_UNSUPPORTED)
    assert b"hidden layers" in lib.neddf_last_error()
    # a skip on the last distance layer would feed 256 + 6 pos channels into the 256-wide heads
    for ddf, extra in ((6, [0]), (3, []), (8, [1, 4])):
        assert codes(ddf_layer_count=ddf, skips=extra + [ddf - 2]) == (NEDDF_E_INVALID, NEDDF_E_INVALID), ddf
        assert b"skip" in lib.neddf_last_error()
    # one layer earlier is accepted (C6 has skips [0, 3] with ddf_layer_count = 6), and so are 24 hidden layers (C7)
    for name in ("C6_fp32_limit", "C7_deepest"):
        cfg = neddf_b200.NeDDF(**fcfg.kwargs(name))._config_struct()
        assert lib.neddf_field_layer_shapes(C.byref(cfg), None, 0) == len(orc.layer_shapes(fcfg.field_config(name)))


def test_table_spans_the_engine_boundaries():
    """The table reaches both sides of each tensor-core bound and the limits it claims to reach."""
    dims = {}
    for name in fcfg.NAMES:
        kw = fcfg.CONFIGS[name]["kw"]
        n_e0 = 6 * kw["embed_pos_rank"]
        off_h = 6 * (kw["embed_pos_rank"] + kw["embed_dir_rank"]) + 3
        dims[name] = (n_e0, off_h, (kw["ddf_layer_count"] - 1) + (kw["col_layer_count"] - 1))
        tc_ok = n_e0 <= 64 and off_h <= 96
        assert tc_ok == ("tc" in fcfg.CONFIGS[name]["engines"]), name
    assert dims["C2_minimal"][:2] == (6, 15)
    assert dims["C3_aux_edge"][1] == 93
    assert dims["C4_past_es"][0] == 66
    assert dims["C5_past_aux"][:2] == (48, 99)
    assert dims["C6_fp32_limit"][1] + 256 + dims["C6_fp32_limit"][0] == 547  # k_total of the fp32 engine
    assert dims["C7_deepest"][2] == 24
    st = fcfg.state("C8_warmup")
    assert (st.lowpass_alpha, st.aux_grad_scale) == (3.5, 0.15)
    s = orc.lowpass_scale(10, st.lowpass_alpha, torch.float64)
    assert float(s[2]) == 1.0 and 0.5 < float(s[3]) < 0.51 and float(s[4:].max()) == 1e-7


def _inputs(name, dtype):
    B, S = 3, 13
    d, o, dists = fcfg.rays(B, S, fcfg.SEED[name] + 3)
    pos, dd, var = orc.cone_samples(d.to(dtype), o.to(dtype), dists.to(dtype), orc.CONE_RAY_RADIUS)
    gd, gc, gp = (t.to(dtype) for t in fcfg.upstream(B, S, fcfg.SEED[name] + 4))
    return pos, dd.contiguous(), var, gd, gc, gp


@pytest.mark.parametrize("name", fcfg.NAMES)
def test_manual_backward_matches_autograd_fp64(name):
    """The derivation of field_bwd.cu (skips at 0 / consecutive / several, no hidden-to-hidden layer, the low-pass
    window, a zero and a missing penalty weight) against autograd, all in fp64."""
    cfg, st = fcfg.field_config(name), fcfg.state(name)
    P = {k: v.double() for k, v in fcfg.params(name).items()}
    pos, dd, var, gd, gc, gp = _inputs(name, torch.float64)
    Pg = {k: v.clone().requires_grad_(True) for k, v in P.items()}
    out = orc.field_forward(Pg, cfg, st, pos, dd, var)
    ((out["density"] * gd).sum() + (out["color"] * gc).sum() + (out["fields_penalty"] * gp).sum()).backward()
    grads = field_backward(P, cfg, st, pos, dd, var, gd, gc, gp)
    assert set(grads) == set(P)
    for k, v in Pg.items():
        assert float(v.grad.abs().max()) > 0.0 or k.endswith(".bias"), k  # every weight is reached
        assert nerr(grads[k].numpy(), v.grad.numpy()) < 1e-7, k


GOLDEN_NAMES = ["C2_minimal", "C7_deepest"]


@pytest.mark.parametrize("name", GOLDEN_NAMES)
def test_oracle_matches_reference_at_other_structures(name):
    """Outputs and parameter gradients of the reference's own NeDDF (tests/golden/make_field_config_golden.py) at the
    seeded parameters: the fp64 oracle reproduces them, so the GPU suite's arbiter is right at these structures."""
    z = np.load(os.path.join(GOLDEN, f"case_cfg_{name}.npz"))
    meta = json.loads(str(z["cfg"]))
    assert meta["kw"] == json.loads(json.dumps(fcfg.kwargs(name))) and meta["iter"] == fcfg.CONFIGS[name]["iter"]
    assert meta["seed"] == fcfg.SEED[name]
    cfg, st = fcfg.field_config(name), fcfg.state(name)
    P = {k: v.double().requires_grad_(True) for k, v in fcfg.params(name).items()}
    t = {k: torch.from_numpy(z[k]).double() for k in ("pos", "dirs", "var", "g_density", "g_color", "g_penalty")}
    out = orc.field_forward(P, cfg, st, t["pos"], t["dirs"], t["var"])
    for k in ("distance", "density", "color", "fields_penalty", "aux_grad"):
        assert_parity(out[k].detach().numpy(), z["out_" + k], 2e-5, fcfg.kinked(name), k)
    ((out["density"] * t["g_density"]).sum() + (out["color"] * t["g_color"]).sum()
     + (out["fields_penalty"] * t["g_penalty"]).sum()).backward()
    for k, v in P.items():
        g = v.grad.numpy()
        g = g[::8, ::4] if (g.ndim == 2 and g.shape[1] > 3) else g
        # the reference runs in fp32: ~1e-6 of fp64 at these depths (measured <= 2e-6)
        assert nerr(g, z["grad_" + k]) < 5e-5, k
