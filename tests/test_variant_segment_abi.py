"""CPU: the refusals of neddf_nerf_forward_rays_segment / neddf_neus_forward_rays_segment return NEDDF_E_INVALID with a
message before any CUDA call (NULL arguments, bad n_edges / sampling_type, a segment outside [0, n_edges), a ray list
without its count or the reverse), so a bad segment never reaches a launch."""
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


def _calls(lib, p, n_edges=9, stype=1, e0=0, seg=2, idx=None, cnt=None, dists=True):
    lp = C.cast(p, C.POINTER(C.c_float))
    d = p if dists else None
    n = C.c_int64(4)
    return {"neddf_nerf_forward_rays_segment": lib.neddf_nerf_forward_rays_segment(p, lp, p, p, d, n, n_edges, stype, 0.0, e0, seg, idx, cnt,
                                                                                   p, p, None),
            "neddf_neus_forward_rays_segment": lib.neddf_neus_forward_rays_segment(p, p, p, d, n, n_edges, stype, 0.0, e0, seg, idx, cnt,
                                                                                   p, p, None)}


def _refused(lib, p, why, **kw):
    for who, rc in _calls(lib, p, **kw).items():
        assert rc == INVALID, (who, kw)
    # the last call's message (each entry point names itself)
    assert lib.neddf_last_error().decode() == f"neddf_neus_forward_rays_segment: {why}", kw


def test_segment_entry_points_refuse_null_arguments(lib, mem):
    p, _ = mem
    _refused(lib, p, "null argument", dists=False)
    lp = C.cast(p, C.POINTER(C.c_float))
    assert lib.neddf_nerf_forward_rays_segment(p, lp, p, p, p, 4, 9, 1, 0.0, 0, 2, None, None, p, None, None) == INVALID
    assert lib.neddf_last_error().decode() == "neddf_nerf_forward_rays_segment: null argument"


@pytest.mark.parametrize("n_edges, stype", [(0, 1), (9, 2)])
def test_segment_entry_points_refuse_bad_edges_or_sampling(lib, mem, n_edges, stype):
    p, _ = mem
    _refused(lib, p, "bad n_edges / sampling_type", n_edges=n_edges, stype=stype)


@pytest.mark.parametrize("e0, seg", [(-1, 2), (0, 0), (0, -3), (8, 2), (9, 1), (0, 10), (2**31 - 1, 1)])
def test_segment_entry_points_refuse_segments_outside_the_rays(lib, mem, e0, seg):
    p, _ = mem
    _refused(lib, p, "bad segment (need 0 <= edge0, 1 <= seg_len, edge0 + seg_len <= n_edges)", e0=e0, seg=seg)


def test_segment_entry_points_refuse_a_ray_list_without_its_count(lib, mem):
    p, _ = mem
    _refused(lib, p, "d_ray_index and d_n_active go together", idx=p)
    _refused(lib, p, "d_ray_index and d_n_active go together", cnt=p)
