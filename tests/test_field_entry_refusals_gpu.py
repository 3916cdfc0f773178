"""H100: every refusal of the seven NeDDF field entry points on samples or rays (neddf_field_forward, _forward_rays,
_forward_rays_segment, _forward_train, _backward, _forward_train_samples, _backward_samples): its return code, its
message, and the order of the checks (each case breaks one argument of an otherwise valid call, or several to pin which
check comes first).  A refused call launches nothing; an empty forward launch succeeds before its pointers and state
are looked at."""
import ctypes as C

import pytest
import torch

from tests import field_configs as fcfg

pytestmark = pytest.mark.gpu

OK, INVALID = 0, -1
POINT, CONE = 0, 1


@pytest.fixture(scope="module")
def env():
    import __graft_entry__ as ge
    ge.build()
    import neddf_b200
    from neddf_b200 import _lib as L
    lib = L.lib()
    name = fcfg.NAMES[0]
    net = neddf_b200.NeDDF(**fcfg.kwargs(name))
    net.load_state_dict(fcfg.params(name))
    net.to("cuda:0")
    h = net._field(torch.device("cuda:0"))
    bare = C.c_void_p()  # a handle whose weights were never set
    cfg = net._config_struct()
    assert lib.neddf_field_create(C.byref(cfg), C.byref(bare)) == OK
    buf = torch.zeros(1 << 12, device="cuda:0")  # non-NULL stand-in for every device pointer: refused calls read none
    torch.cuda.synchronize()
    yield lib, h, bare, net._state_struct(), buf.data_ptr()
    lib.neddf_field_destroy(bare)


def _args(env, entry, **kw):
    """A valid call of `entry` (4 samples or 4 rays of 9 edges, cone sampling) with the arguments in kw replaced."""
    lib, h, _, st, p = env
    a = dict(f=h, st=C.byref(st), pos=p, dir=p, var=p, n=4, ray_dir=p, ray_orig=p, dists=p, n_rays=4, n_edges=9,
             stype=CONE, edge0=0, seg_len=2, ray_index=None, n_active=None, save_pre=p, g_density=p, g_color=p, g_penalty=p,
             post=p, gpre=p, ghead_da=p, ghead_col=p, xes=p, xcol=p, density=p, color=p)
    a.update(kw)
    rays = (a["f"], a["st"], a["ray_dir"], a["ray_orig"], a["dists"], a["n_rays"], a["n_edges"], a["stype"], 0.01)
    samples = (a["f"], a["st"], a["pos"], a["dir"], a["var"], a["n"])
    bwd = (a["save_pre"], a["g_density"], a["g_color"], a["g_penalty"], a["post"], a["gpre"], a["ghead_da"], a["ghead_col"],
           a["xes"], a["xcol"], None)
    return {
        "neddf_field_forward": samples + (p, a["density"], a["color"], p, p, 0, 0, None),
        "neddf_field_forward_rays": rays + (p, a["density"], a["color"], p, p, 0, 0, None),
        "neddf_field_forward_rays_segment": rays + (a["edge0"], a["seg_len"], a["ray_index"], a["n_active"], a["density"],
                                                    a["color"], 0, None),
        "neddf_field_forward_train": rays + (a["density"], a["color"], p, a["save_pre"], 0, None),
        "neddf_field_backward": rays + bwd,
        "neddf_field_forward_train_samples": samples + (p, a["density"], a["color"], p, p, a["save_pre"], 0, None),
        "neddf_field_backward_samples": samples + bwd,
    }[entry]


def _call(env, entry, **kw):
    lib = env[0]
    before = lib.neddf_launch_count()
    rc = getattr(lib, entry)(*_args(env, entry, **kw))
    assert lib.neddf_launch_count() == before, (entry, kw)
    return rc, lib.neddf_last_error().decode()


SAMPLES = ("neddf_field_forward", "neddf_field_forward_train_samples", "neddf_field_backward_samples")
RAYS = ("neddf_field_forward_rays", "neddf_field_forward_rays_segment", "neddf_field_forward_train", "neddf_field_backward")
TRAIN = SAMPLES[1:] + RAYS[2:]
BAD_STATE = {"lowpass_alpha": -1.0}  # outside [0, embed_pos_rank): refused by the state checks
UNNAMED = {"field state is NULL", "lowpass_alpha out of range"}  # the state checks' messages name no entry point


def _st(env, **fields):
    st = type(env[3]).from_buffer_copy(env[3])
    for k, v in fields.items():
        setattr(st, k, v)
    return C.byref(st)


def _cases(env):
    _, _, bare, _, p = env
    null = None
    c = []  # (entry, arguments, message after "<entry>: ")
    for e in SAMPLES + RAYS:
        c += [(e, dict(f=null, n_edges=0, stype=7, pos=null, ray_dir=null, st=null), "field is NULL"),
              (e, dict(f=bare, n=-1, n_rays=-1, pos=null, ray_dir=null, st=null), "weights were never set"),
              (e, dict(st=null), "field state is NULL"),
              (e, dict(st=_st(env, **BAD_STATE)), "lowpass_alpha out of range")]
    for e in SAMPLES:
        empty = "n < 0" if e == "neddf_field_forward" else "n <= 0"
        c += [(e, dict(n=-1, pos=null, st=null), empty),
              (e, dict(pos=null, st=null), "NULL input pointer"),
              (e, dict(dir=null), "NULL input pointer"),
              (e, dict(var=null), "NULL input pointer")]
        if e != "neddf_field_forward":
            c += [(e, dict(n=0, pos=null, st=null), "n <= 0")]
    for e in RAYS:
        null_msg = "NULL pointer" if e == "neddf_field_forward_rays_segment" else "NULL input pointer"
        c += [(e, dict(n_rays=-1, stype=7, ray_dir=null), "bad sizes"),
              (e, dict(n_edges=0, stype=7), "bad sizes"),
              (e, dict(stype=7, n_edges=1, seg_len=1, ray_dir=null), "unknown sampling type"),
              (e, dict(stype=CONE, n_edges=1, edge0=0, seg_len=1, ray_dir=null), "cone sampling needs >= 2 edges"),
              (e, dict(ray_dir=null, st=null), null_msg),
              (e, dict(ray_orig=null), null_msg),
              (e, dict(dists=null), null_msg)]
        if e in TRAIN:
            c += [(e, dict(n_rays=0, ray_dir=null, st=null), "bad sizes")]
    seg = "neddf_field_forward_rays_segment"
    for e0, n in [(-1, 2), (0, 0), (0, -3), (8, 2), (9, 1), (0, 10)]:
        c += [(seg, dict(edge0=e0, seg_len=n, stype=7, ray_dir=null), "bad sizes")]
    c += [(seg, dict(density=null, st=null), "NULL pointer"),
          (seg, dict(color=null), "NULL pointer"),
          (seg, dict(ray_index=p, st=null), "d_ray_index and d_n_active go together"),
          (seg, dict(n_active=p), "d_ray_index and d_n_active go together")]
    for e in TRAIN:
        if e.endswith(("forward_train", "forward_train_samples")):
            c += [(e, dict(save_pre=null), "d_save_pre is NULL")]
        else:
            c += [(e, dict(**{b: null}), "NULL buffer")
                  for b in ("save_pre", "g_density", "g_color", "post", "gpre", "ghead_da", "ghead_col", "xes", "xcol")]
    return c


def test_field_entry_points_refuse_each_bad_argument_in_order(env):
    n = 0
    for entry, kw, why in _cases(env):
        rc, msg = _call(env, entry, **kw)
        assert (rc, msg) == (INVALID, why if why in UNNAMED else f"{entry}: {why}"), (entry, kw)
        n += 1
    assert n > 100


@pytest.mark.parametrize("entry", ["neddf_field_forward", "neddf_field_forward_rays", "neddf_field_forward_rays_segment"])
def test_empty_forward_is_a_no_op_before_pointers_and_state(env, entry):
    assert _call(env, entry, n=0, n_rays=0, pos=None, dir=None, var=None, ray_dir=None, ray_orig=None, dists=None, st=None,
                 density=None, color=None)[0] == OK


def test_segment_bound_is_checked_without_int32_overflow(env):
    """edge0 + seg_len past INT32_MAX is outside the rays like any other segment end past n_edges."""
    seg = "neddf_field_forward_rays_segment"
    assert _call(env, seg, edge0=2**31 - 1, seg_len=1) == (INVALID, f"{seg}: bad sizes")
    assert _call(env, seg, edge0=1, seg_len=2**31 - 1) == (INVALID, f"{seg}: bad sizes")
