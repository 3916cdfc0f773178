"""CPU: the C-ABI shared library loads and exports every symbol include/neddf_b200.h declares
(no compute calls - there is no GPU in the build container)."""
import ctypes
import os
import re

import pytest


@pytest.fixture(scope="module")
def built(repo_root):
    import __graft_entry__ as ge
    ge.build()
    return os.path.join(repo_root, "neddf_b200", "libneddf_b200.so")


def _declared(repo_root):
    src = open(os.path.join(repo_root, "include", "neddf_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(neddf_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol(repo_root, built):
    lib = ctypes.CDLL(built)
    names = _declared(repo_root)
    assert len(names) >= 17
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/neddf_b200.h but not exported"


def test_python_binding_covers_header(repo_root, built):
    from neddf_b200 import _lib as L
    assert L.exported_symbols() == _declared(repo_root)
    lib = L.lib()
    assert lib.neddf_abi_version() == 3
    assert lib.neddf_launch_count() == 0


def test_layer_shapes_and_validation(built):
    import ctypes as C

    import neddf_b200
    from neddf_b200 import _lib as L
    from oracle import neddf_oracle as orc
    lib = L.lib()
    for kw in (dict(col_layer_count=4), dict(), dict(ddf_layer_count=6, skips=[2]), dict(skips=[1, 4])):
        net = neddf_b200.NeDDF(**kw)
        cfg = net._config_struct()
        buf = (C.c_int32 * 96)()
        n = lib.neddf_field_layer_shapes(C.byref(cfg), buf, 48)
        ref = orc.layer_shapes(orc.FieldConfig(**kw))
        assert n == len(ref)
        assert [(buf[2 * i], buf[2 * i + 1]) for i in range(n)] == [(a, b) for _, a, b in ref]
        # module parameter shapes are the reference's (weight stored [in,out])
        sd = net.state_dict()
        for name, a, b in ref:
            assert tuple(sd[name + ".weight"].shape) == (a, b) and tuple(sd[name + ".bias"].shape) == (b,)
    bad = neddf_b200.NeDDF(ddf_layer_width=128, col_layer_width=128)
    cfg = bad._config_struct()
    assert lib.neddf_field_layer_shapes(C.byref(cfg), None, 0) == -3  # NEDDF_E_UNSUPPORTED
    assert b"256" in lib.neddf_last_error()


def test_nerf_structure_limits_are_refused_before_any_launch(built):
    """The configuration checks of the two NeRF handles at their boundaries.  A refused structure returns the code its
    entry point has always returned, before any CUDA call.  An accepted one gets as far as allocating its packed weights
    (NEDDF_OK with a GPU, NEDDF_E_CUDA without one).  neddf_nerf_layer_shapes checks the layer count only."""
    import ctypes as C

    from neddf_b200 import _lib as L
    lib = L.lib()
    OK, INVALID, CUDA, UNSUPPORTED = 0, -1, -2, -3
    accepted = (OK, CUDA)

    def cfg(layer_count=8, pos=10, dirs=4, skips=(4,), act=1, density_act=1):
        c = L.NerfConfig()
        c.embed_pos_rank, c.embed_dir_rank, c.layer_count, c.layer_width = pos, dirs, layer_count, 256
        c.activation_type, c.density_activation_type = act, density_act
        c.n_skips = len(skips)
        for i, v in enumerate(skips):
            c.skips[i] = v
        return c

    def codes(**kw):
        c = cfg(**kw)
        out = [lib.neddf_nerf_layer_shapes(C.byref(c), None, 0)]
        for create, destroy in ((lib.neddf_nerf_create, lib.neddf_nerf_destroy),
                                (lib.neddf_nerf_train_create, lib.neddf_nerf_train_destroy)):
            h = C.c_void_p()
            rc = create(C.byref(c), C.byref(h))
            assert (rc == OK) == bool(h.value)
            if h.value:
                destroy(h)
            out.append("accepted" if rc in accepted else rc)
        return tuple(out)

    # layer_count: forward 2..13, training backward 2..12
    assert codes(layer_count=1, skips=()) == (INVALID, UNSUPPORTED, UNSUPPORTED)
    assert codes(layer_count=2, skips=()) == (5, "accepted", "accepted")
    assert codes(layer_count=12) == (15, "accepted", "accepted")
    assert codes(layer_count=13) == (16, "accepted", UNSUPPORTED)
    assert b"2..12" in lib.neddf_last_error()
    assert codes(layer_count=14) == (INVALID, UNSUPPORTED, UNSUPPORTED)
    assert b"2..12" in lib.neddf_last_error()
    c = cfg(layer_count=14)
    assert lib.neddf_nerf_create(C.byref(c), C.byref(C.c_void_p())) == UNSUPPORTED
    assert b"layer_count must be 2..13" in lib.neddf_last_error()
    # embedding ranks: 6 * embed_pos_rank <= 64, 6 * embed_dir_rank <= 32
    assert codes(pos=10) == (11, "accepted", "accepted")
    assert codes(pos=11) == (11, UNSUPPORTED, UNSUPPORTED)
    assert codes(dirs=5) == (11, "accepted", "accepted")
    assert codes(dirs=6) == (11, UNSUPPORTED, UNSUPPORTED)
    # a skip after the last hidden layer would widen the heads
    assert codes(skips=(6,)) == (11, "accepted", "accepted")
    assert codes(skips=(7,)) == (11, UNSUPPORTED, UNSUPPORTED)
    assert b"skip" in lib.neddf_last_error()
    # activation ids: a malformed one is an invalid argument to the forward
    for kw in (dict(act=3), dict(density_act=-1)):
        assert codes(**kw) == (11, INVALID, UNSUPPORTED), kw
        assert b"bad activation" in lib.neddf_last_error()


def test_entry_points_fail_loudly_without_a_gpu(built):
    """No CPU fallback: with no CUDA device (this container) creating a field returns an error code
    and a message, NULL arguments are rejected before any CUDA call, nothing crashes or leaks a handle."""
    import ctypes as C

    import torch

    import neddf_b200
    from neddf_b200 import _lib as L
    lib = L.lib()
    assert lib.neddf_field_create(None, None) < 0 and lib.neddf_last_error()
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    cfg = neddf_b200.NeDDF()._config_struct()
    handle = C.c_void_p()
    rc = lib.neddf_field_create(C.byref(cfg), C.byref(handle))
    assert rc < 0 and not handle.value
    assert b"CUDA" in lib.neddf_last_error() or b"cuda" in lib.neddf_last_error()
    assert lib.neddf_field_destroy(None) in (0, -1, -2)  # tolerated, never a crash
    with pytest.raises(Exception):  # the Python surface refuses CPU tensors instead of computing on the host
        neddf_b200.NeDDF()(neddf_b200.Sampling(torch.zeros(1, 2, 3), torch.zeros(1, 2, 3), torch.zeros(1, 2, 3)))
