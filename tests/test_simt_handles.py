"""CPU: the refusals of the four CUDA-core network handles (NeRF, NeRF training, NeuS, NeuS training) that return before
any CUDA call - NULL arguments and bad n_edges / sampling_type - keep their return codes and neddf_last_error()
strings.  The handles share one lifecycle (csrc/simt_tile.cuh), and each entry point keeps its own checks and words."""
import ctypes as C

import pytest

INVALID = -1


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from neddf_b200 import _lib as L
    return L.lib()


@pytest.fixture(scope="module")
def mem():
    """Non-NULL stand-ins for a handle and device pointers: refused calls must not read them."""
    buf = C.create_string_buffer(1 << 16)
    return C.cast(buf, C.c_void_p), buf


def _refuses(lib, rc, msg):
    assert rc == INVALID
    assert lib.neddf_last_error().decode() == msg


def test_create_and_set_weights_refuse_null_arguments(lib, mem):
    from neddf_b200 import _lib as L
    p, _ = mem
    out = C.c_void_p()
    nerf_cfg, neus_cfg = L.NerfConfig(), L.NeusConfig()
    _refuses(lib, lib.neddf_nerf_create(None, C.byref(out)), "neddf_nerf_create: null argument")
    _refuses(lib, lib.neddf_nerf_create(C.byref(nerf_cfg), None), "neddf_nerf_create: null argument")
    _refuses(lib, lib.neddf_nerf_train_create(None, C.byref(out)), "neddf_nerf_train_create: null argument")
    _refuses(lib, lib.neddf_nerf_train_create(C.byref(nerf_cfg), None), "neddf_nerf_train_create: null argument")
    _refuses(lib, lib.neddf_neus_create(None, C.byref(out)), "neddf_neus_create: null config")
    _refuses(lib, lib.neddf_neus_create(C.byref(neus_cfg), None), "neddf_neus_create: null argument")
    _refuses(lib, lib.neddf_neus_train_create(None, C.byref(out)), "neddf_neus_train_create: null argument")
    _refuses(lib, lib.neddf_neus_train_create(C.byref(neus_cfg), None), "neddf_neus_train_create: null argument")
    assert out.value is None
    ptrs = (C.c_void_p * 4)()
    for name in ("nerf", "nerf_train"):
        fn = getattr(lib, f"neddf_{name}_set_weights")
        _refuses(lib, fn(None, ptrs, ptrs, 11, None), f"neddf_{name}_set_weights: null argument")
        _refuses(lib, fn(p, None, ptrs, 11, None), f"neddf_{name}_set_weights: null argument")
    for name in ("neus", "neus_train"):
        fn = getattr(lib, f"neddf_{name}_set_weights")
        _refuses(lib, fn(None, ptrs, ptrs, 11, p, None), f"neddf_{name}_set_weights: null argument")
        _refuses(lib, fn(p, ptrs, ptrs, 11, None, None), f"neddf_{name}_set_weights: null argument")


def test_forward_and_backward_refuse_null_arguments(lib, mem):
    p, _ = mem
    lp = C.cast(p, C.POINTER(C.c_float))
    bufs = (C.c_void_p * 9)(*([p] * 9))
    n = C.c_int64(64)
    _refuses(lib, lib.neddf_nerf_forward(None, lp, p, p, p, n, p, p, None), "neddf_nerf_forward: null argument")
    _refuses(lib, lib.neddf_nerf_forward(p, lp, p, p, None, n, p, p, None), "neddf_nerf_forward: null argument")
    _refuses(lib, lib.neddf_nerf_forward_rays(p, lp, p, p, None, n, 65, 1, 0.0, p, p, None), "neddf_nerf_forward_rays: null argument")
    _refuses(lib, lib.neddf_nerf_train_backward(None, lp, p, p, p, n, *([p] * 9), None), "neddf_nerf_train_backward: null argument")
    _refuses(lib, lib.neddf_nerf_train_backward(p, lp, p, p, None, n, *([p] * 9), None), "neddf_nerf_train_backward: null argument")
    _refuses(lib, lib.neddf_nerf_train_backward_rays(p, lp, p, p, None, n, 65, 1, 0.0, *([p] * 9), None),
             "neddf_nerf_train_backward_rays: null argument")
    _refuses(lib, lib.neddf_neus_forward(None, p, p, n, p, p, p, None, None), "neddf_neus_forward: null argument")
    _refuses(lib, lib.neddf_neus_forward(p, p, p, n, p, p, None, None, None), "neddf_neus_forward: null argument")
    _refuses(lib, lib.neddf_neus_forward_rays(p, p, p, None, n, 65, 1, 0.0, p, p, p, None, None), "neddf_neus_forward_rays: null argument")
    _refuses(lib, lib.neddf_neus_train_backward(None, p, p, n, None, p, p, None, bufs, None), "neddf_neus_train_backward: null argument")
    _refuses(lib, lib.neddf_neus_train_backward(p, p, p, n, None, p, p, None, None, None), "neddf_neus_train_backward: null argument")
    _refuses(lib, lib.neddf_neus_train_backward_rays(p, p, None, p, n, 65, 1, 0.0, None, p, p, None, bufs, None),
             "neddf_neus_train_backward_rays: null argument")


@pytest.mark.parametrize("n_edges, sampling_type", [(0, 1), (-3, 0), (65, 2), (65, -1)])
def test_rays_entry_points_refuse_bad_edges_or_sampling(lib, mem, n_edges, sampling_type):
    p, _ = mem
    lp = C.cast(p, C.POINTER(C.c_float))
    bufs = (C.c_void_p * 9)(*([p] * 9))
    n = C.c_int64(4)
    _refuses(lib, lib.neddf_nerf_forward_rays(p, lp, p, p, p, n, n_edges, sampling_type, 0.0, p, p, None),
             "neddf_nerf_forward_rays: bad n_edges / sampling_type")
    _refuses(lib, lib.neddf_nerf_train_backward_rays(p, lp, p, p, p, n, n_edges, sampling_type, 0.0, *([p] * 9), None),
             "neddf_nerf_train_backward_rays: bad n_edges / sampling_type")
    _refuses(lib, lib.neddf_neus_forward_rays(p, p, p, p, n, n_edges, sampling_type, 0.0, p, p, p, None, None),
             "neddf_neus_forward_rays: bad n_edges / sampling_type")
    _refuses(lib, lib.neddf_neus_train_backward_rays(p, p, p, p, n, n_edges, sampling_type, 0.0, None, p, p, None, bufs, None),
             "neddf_neus_train_backward_rays: bad n_edges / sampling_type")
