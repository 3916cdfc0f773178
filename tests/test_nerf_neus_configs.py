"""CPU: the NeRF and NeuS structures of tests/nerf_neus_configs.py on the host side - the C ABI's layer tables against the
oracle and the modules, which handles accept each structure, and the NeuS configuration check at its boundaries."""
import ctypes as C

import pytest

from tests import nerf_neus_configs as ncfg

OK, INVALID, CUDA, UNSUPPORTED = 0, -1, -2, -3
ACCEPTED = (OK, CUDA)  # an accepted structure gets as far as allocating its packed weights (NEDDF_E_CUDA without a GPU)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from neddf_b200 import _lib as L
    return L.lib()


def _module(name):
    import neddf_b200
    return (neddf_b200.NeRF if ncfg.variant(name) == "nerf" else neddf_b200.NeuS)(**ncfg.kwargs(name))


def _create(lib, prefix, cfg):
    """Return code of <prefix>_create; a handle it made is destroyed again."""
    h = C.c_void_p()
    rc = getattr(lib, prefix + "_create")(C.byref(cfg), C.byref(h))
    assert (rc == OK) == bool(h.value)
    if h.value:
        getattr(lib, prefix + "_destroy")(h)
    return rc


@pytest.mark.parametrize("name", ncfg.NAMES)
def test_layer_table_matches_oracle_and_module(lib, name):
    net = _module(name)
    cfg = net._config_struct()
    buf = (C.c_int32 * 128)()
    n = getattr(lib, f"neddf_{ncfg.variant(name)}_layer_shapes")(C.byref(cfg), buf, 64)
    ref = ncfg.layer_shapes(name)
    assert n == len(ref) == len(net._ordered_layers())
    assert [(buf[2 * i], buf[2 * i + 1]) for i in range(n)] == [(a, b) for _, a, b in ref]
    sd = net.state_dict()
    extra = {"variance"} if ncfg.variant(name) == "neus" else set()
    assert set(sd) == {f"{k}.{p}" for k, _, _ in ref for p in ("weight", "bias")} | extra
    for k, a, b in ref:  # torch Linear layout: weight [out, in]
        assert tuple(sd[k + ".weight"].shape) == (b, a) and tuple(sd[k + ".bias"].shape) == (b,), k
    net.load_state_dict(ncfg.state_dict(name))  # strict: the seeded parameters fit the module exactly


@pytest.mark.parametrize("name", ncfg.NAMES)
def test_handles_accept_what_the_table_says(lib, name):
    """Every entry is accepted by the forward handle; the training handle refuses exactly the entries marked so, with
    the limit in its message."""
    cfg = _module(name)._config_struct()
    v = ncfg.variant(name)
    assert _create(lib, f"neddf_{v}", cfg) in ACCEPTED
    rc = _create(lib, f"neddf_{v}_train", cfg)
    if ncfg.CONFIGS[name]["train"]:
        assert rc in ACCEPTED
    else:
        assert rc == UNSUPPORTED and b"2..12" in lib.neddf_last_error()


def test_table_reaches_the_limits_it_claims():
    k = {n: ncfg.CONFIGS[n]["kw"] for n in ncfg.NAMES}
    assert (6 * k["N2_max_embed"]["embed_pos_rank"], 6 * k["N2_max_embed"]["embed_dir_rank"]) == (60, 30)
    assert k["N3_deep_fwd"]["layer_count"] == 13 and max(k["N3_deep_fwd"]["skips"]) == 13 - 2
    assert k["N4_deep_train"]["layer_count"] == 12
    assert len(k["N5_eight_skips"]["skips"]) == len(k["S4_eight_skips"]["skips"]) == 8
    assert ncfg.lowpass_alpha("N6_warmup") == 3.5
    assert k["S1_one_sdf"]["sdf_layer_count"] == 1
    assert 6 + 6 * k["S2_max_embed"]["embed_dir_rank"] == 30
    assert (k["S3_deepest"]["sdf_layer_count"], k["S3_deepest"]["col_layer_count"]) == (12, 12)
    assert max(k["S3_deepest"]["skips"]) == 12 - 2
    assert {k: a for k, a, _ in ncfg.layer_shapes("S2_max_embed")}["layers_col.0"] == 286
    assert {k: a for k, a, _ in ncfg.layer_shapes("N2_max_embed")}["layers.1"] == 316


def test_sharp_entry_spans_the_density_underflow():
    """S5: the seeded sdf reaches tanhExp's floor and passes the point where fp32's exp(-20 sdf) underflows to 0."""
    import torch

    from oracle import neddf_oracle as orc
    P = ncfg.params("S5_sharp")
    pos, dirs, _ = ncfg.samples(1, 2000, 1)
    out = orc.neus_forward(P, ncfg.config("S5_sharp"), pos, dirs)
    assert float(out["sdf"].min()) < -0.34 and float(out["sdf"].max()) > 5.0
    zero = orc.neus_density(out["sdf"].float(), P["variance"].float()) == 0
    assert 0.1 < float(zero.float().mean()) < 0.5 and bool(torch.isfinite(out["density"]).all())


def test_neus_structure_limits_are_refused_before_any_launch(lib):
    """The configuration check shared by neddf_neus_layer_shapes and both NeuS handles, at its boundaries."""
    from neddf_b200 import _lib as L
    ids = L.ACT_IDS

    def cfg(sdf=8, col=8, pos=6, dirs=4, skips=(4,), act="ReLU", n_skips=None):
        c = L.NeusConfig()
        c.embed_pos_rank, c.embed_dir_rank = pos, dirs
        c.sdf_layer_count, c.sdf_layer_width, c.col_layer_count, c.col_layer_width = sdf, 256, col, 256
        c.activation_type = ids[act]
        c.n_skips = len(skips) if n_skips is None else n_skips
        for i, v in enumerate(skips):
            c.skips[i] = v
        return c

    def codes(**kw):
        c = cfg(**kw)
        out = [lib.neddf_neus_layer_shapes(C.byref(c), None, 0)]
        for prefix in ("neddf_neus", "neddf_neus_train"):
            rc = _create(lib, prefix, c)
            out.append("accepted" if rc in ACCEPTED else rc)
        return tuple(out)

    refused = (UNSUPPORTED, UNSUPPORTED, UNSUPPORTED)
    # trunk depths 1..12
    assert codes(sdf=1, skips=()) == (1 + 8 + 1, "accepted", "accepted")
    assert codes(sdf=12) == (12 + 8 + 1, "accepted", "accepted")
    assert codes(col=1) == (8 + 1 + 1, "accepted", "accepted")
    assert codes(col=12) == (8 + 12 + 1, "accepted", "accepted")
    for kw, what in ((dict(sdf=0, skips=()), b"sdf_layer_count"), (dict(sdf=13), b"sdf_layer_count"),
                     (dict(col=0), b"col_layer_count"), (dict(col=13), b"col_layer_count")):
        assert codes(**kw) == refused, kw
        assert what in lib.neddf_last_error() and b"1..12" in lib.neddf_last_error()
    # embeddings: 6 * embed_pos_rank <= 64, 6 + 6 * embed_dir_rank <= 32
    assert codes(pos=10) == (17, "accepted", "accepted")
    assert codes(pos=11) == refused
    assert codes(dirs=4) == (17, "accepted", "accepted")
    assert codes(dirs=5) == refused
    assert b"embed_dir_rank" in lib.neddf_last_error()
    # a skip on the last SDF layer; one layer earlier is accepted
    assert codes(sdf=6, skips=(0, 4)) == (6 + 8 + 1, "accepted", "accepted")
    for sdf, skips in ((6, (0, 5)), (1, (0,)), (12, (11,))):
        assert codes(sdf=sdf, skips=skips) == refused, (sdf, skips)
        assert b"skip" in lib.neddf_last_error()
    assert codes(sdf=12, skips=tuple(range(8))) == (12 + 8 + 1, "accepted", "accepted")
    assert codes(sdf=12, skips=tuple(range(8)), n_skips=9) == refused
    assert b"8 skips" in lib.neddf_last_error()
    # NeuS takes ReLU and tanhExp only (the reference's activation dictionary)
    assert codes(act="tanhExp") == (17, "accepted", "accepted")
    assert codes(act="LeakyReLU") == refused
    assert b"activation_type" in lib.neddf_last_error()
    import neddf_b200
    with pytest.raises(KeyError):
        neddf_b200.NeuS(activation_type="LeakyReLU")
