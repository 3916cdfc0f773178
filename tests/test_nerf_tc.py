"""CPU: the NeRF tensor-core engine (csrc/nerf_tc.cu behind neddf_nerf_tc_*) without a GPU - its precision model on the
oracle, the configurations its handle refuses, and how neddf_b200.NeRF picks a kernel per engine over a fake library."""
import contextlib
import ctypes as C

import pytest
import torch

import neddf_b200
from neddf_b200 import _lib as L
from neddf_b200._host import KernelHandle
from neddf_b200.network import BaseNeuralField, EngineRangeError
from neddf_b200.ray import Sampling
from oracle import neddf_oracle as orc
from tests import nerf_neus_configs as ncfg
from tests.field_configs import samples
from tests.helpers import PARITY_TOL, nerr
from tests.test_field_host_glue import FakeLib
from tests.test_nerf_oracle import NerfCase


def nerf_forward_mm(P, cfg, lowpass_alpha, pos, dirs, var, mm):
    """orc.nerf_forward with the kernel's GEMMs (hidden layers and outL_color.0) as ``mm`` (orc.split_matmul); the
    density and colour heads stay plain fp32 products, as in the kernel."""
    B, S = pos.shape[0], pos.shape[1]
    n = B * S
    x3, d3, v3 = pos.reshape(n, 3), dirs.reshape(n, 3), var.reshape(n, 3)
    E = cfg.embed_pos_rank
    scale = orc.lowpass_scale(E, lowpass_alpha, pos.dtype).reshape(1, E, 1).expand(1, E, 3).reshape(1, 3 * E)
    scale = scale * orc.pe_weights(v3, E)
    embed_pos = orc.pe_plain(x3, E) * torch.cat([scale, scale], 1)
    embed_dir = orc.pe_plain(d3, cfg.embed_dir_rank)
    act = {"ReLU": torch.relu, "LeakyReLU": torch.nn.functional.leaky_relu,
           "tanhExp": lambda t: orc.density_act("tanhExp", t)}[cfg.activation_type]
    hx = embed_pos
    for lid in range(cfg.layer_count):
        hx = act(mm(hx, P[f"layers.{lid}.weight"]) + P[f"layers.{lid}.bias"])
        if lid in cfg.skips:
            hx = torch.cat([hx, embed_pos], 1)
    density = orc.density_act(cfg.density_activation_type, hx @ P["outL_density.weight"] + P["outL_density.bias"])
    c1 = torch.relu(mm(torch.cat([hx, embed_dir], 1), P["outL_color.0.weight"]) + P["outL_color.0.bias"])
    color = c1 @ P["outL_color.2.weight"] + P["outL_color.2.bias"]
    return {"density": density.reshape(B, S), "color": color.reshape(B, S, 3)}


def _model_cases():
    """(name, params, cfg, alpha, pos, dirs, var): both real-reference goldens on their fine samples, N1-N6 on
    seeded samples."""
    for name in ("relu", "tanhexp"):
        c = NerfCase(name)
        d, o = orc.make_rays(c.t("uv"), c.cam)
        pos, dd, var = orc.make_samples(c.rc, d, o, c.t("dists_fine"))
        yield "case_nerf_" + name, c.params("fine"), c.nc, c.alpha, pos, dd.contiguous(), var
    for name in ncfg.NERF:
        pos, dd, var = samples(4, 256, ncfg.SEED[name])
        yield name, ncfg.params(name), ncfg.config(name), ncfg.lowpass_alpha(name), pos, dd, var


def test_split_fp16_precision_model_meets_a_tenth_of_the_parity_bound():
    """Three fp16 products (hi*hi + lo*hi + hi*lo) stay within 0.1 x PARITY_TOL of the fp32 oracle on every structure,
    N6's subnormal embeddings included; one product (hi*hi) does not, which shows the bar can fail."""
    three, one = orc.split_matmul("fp16", 3), orc.split_matmul("fp16", 1)
    one_fails = []
    for name, P, cfg, alpha, pos, dd, var in _model_cases():
        with torch.no_grad():
            ref = orc.nerf_forward(P, cfg, alpha, pos, dd, var)
            got = nerf_forward_mm(P, cfg, alpha, pos, dd, var, three)
            low = nerf_forward_mm(P, cfg, alpha, pos, dd, var, one)
        for k in ("density", "color"):
            e = nerr(got[k].numpy(), ref[k].numpy())
            assert e < 0.1 * PARITY_TOL, (name, k, e)
        one_fails.append(max(nerr(low[k].numpy(), ref[k].numpy()) for k in ("density", "color")) >= 0.1 * PARITY_TOL)
    assert all(one_fails), one_fails


def test_tc_handle_refuses_exactly_what_the_fp32_handle_refuses(built_lib):
    """neddf_nerf_tc_create at the boundaries test_abi walks for the two CUDA-core NeRF handles: the same code as
    neddf_nerf_create for every structure, refusals before any CUDA call (accepted ones get as far as allocating:
    NEDDF_OK with a GPU, NEDDF_E_CUDA without one)."""
    lib = L.lib()
    OK, CUDA = 0, -2

    def cfg(layer_count=8, pos=10, dirs=4, skips=(4,), act=1, density_act=1):
        c = L.NerfConfig()
        c.embed_pos_rank, c.embed_dir_rank, c.layer_count, c.layer_width = pos, dirs, layer_count, 256
        c.activation_type, c.density_activation_type = act, density_act
        c.n_skips = len(skips)
        for i, v in enumerate(skips):
            c.skips[i] = v
        return c

    def code(create, destroy, c):
        h = C.c_void_p()
        rc = create(C.byref(c), C.byref(h))
        assert (rc == OK) == bool(h.value)
        if h.value:
            destroy(h)
        return "accepted" if rc in (OK, CUDA) else (rc, lib.neddf_last_error().split(b": ", 1)[1])

    structures = [dict(layer_count=n, skips=()) for n in (1, 2, 13, 14)] + [dict(layer_count=12)]
    structures += [dict(pos=p) for p in (0, 1, 10, 11, 17)] + [dict(dirs=d) for d in (0, 1, 5, 6)]
    structures += [dict(skips=s) for s in ((6,), (7,), (0, 1, 2, 3, 4, 5, 6, 7))]
    structures += [dict(act=3), dict(density_act=-1), dict(act=0), dict(act=2, density_act=0)]
    refused = 0
    for kw in structures:
        c = cfg(**kw)
        want = code(lib.neddf_nerf_create, lib.neddf_nerf_destroy, c)
        got = code(lib.neddf_nerf_tc_create, lib.neddf_nerf_tc_destroy, c)
        assert got == want, (kw, got, want)
        refused += want != "accepted"
    assert refused >= 8
    assert lib.neddf_nerf_tc_create(None, None) == -1
    lib.neddf_nerf_tc_destroy(None)  # tolerated


@pytest.fixture
def built_lib(repo_root):
    import __graft_entry__ as ge
    ge.build()


@pytest.fixture
def fake(monkeypatch):
    """FakeLib on CPU tensors; neddf_nerf_tc_status reports (and clears) the word set in ``lib.status``."""
    lib = FakeLib()
    lib.status = {}

    def status(h, out, stream):
        lib.calls.append(("neddf_nerf_tc_status", h.value))
        out._obj.value = lib.status.pop(h.value, 0)
        return 0

    lib.neddf_nerf_tc_status = status
    monkeypatch.setattr(L, "lib", lambda: lib)
    monkeypatch.setattr(L, "stream_ptr", lambda device=None: None)
    monkeypatch.setattr(L, "require_cuda_f32", lambda t, name: t.to(torch.float32).contiguous())
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    # CPU tensors: the forward handles' CUDA-only check is the one thing bypassed
    monkeypatch.setattr(BaseNeuralField, "_field", lambda self, device, kind=0: self._HANDLES[kind].get(self, device))
    seen, get = [], KernelHandle.get

    def tracked_get(kh, net, device):
        seen.append((kh, net))
        return get(kh, net, device)

    monkeypatch.setattr(KernelHandle, "get", tracked_get)
    yield lib
    for kh, net in seen:  # fake handles must never reach the real library's destroy (module __del__ after the test)
        kh.reset(net)


_ENTRIES = ("_forward", "_forward_rays", "_forward_rays_segment")


def _forward_calls(lib):
    """ABI prefix of every forward call recorded since the last clear."""
    out = []
    for c in lib.calls:
        for e in _ENTRIES:
            for pre in ("neddf_nerf_tc", "neddf_nerf"):
                if c[0] == pre + e:
                    out.append((pre, e))
    return out


def _run_all(net):
    """One call of each inference entry point; the prefixes they went to."""
    pos, dd, var = samples(2, 5, 1)
    net.forward(Sampling(pos, dd, var))
    d, o = torch.zeros(2, 3), torch.zeros(2, 3)
    dists = torch.linspace(2, 6, 5).repeat(2, 1)
    net.forward_rays(d, o, dists, "point", 0.0)
    dens, col = torch.zeros(2, 5), torch.zeros(2, 5, 3)
    net.forward_rays_segment(d, o, dists, "point", 0.0, 0, 2, None, None, dens, col)


def _render():
    torch.manual_seed(0)
    return neddf_b200.NeRFRender(network_config={"_target_": "neddf.network.NeRF", "embed_pos_rank": 3, "embed_dir_rank": 2,
                                                 "layer_count": 3, "skips": [0]}, use_coarse_network=True)


def test_engine_selects_the_kernel(fake):
    """The default and "tc2" run neddf_nerf_*; "tc" and "auto" run neddf_nerf_tc_*, on a handle of their own that is
    packed, re-packed and released like the fp32 one."""
    r = _render()
    net = r.network_fine
    assert net.engine == "fp32" and net.resolved_engine() == "fp32"
    with torch.no_grad():
        for engine, pre in (("fp32", "neddf_nerf"), ("tc2", "neddf_nerf"), ("tc", "neddf_nerf_tc"), ("auto", "neddf_nerf_tc")):
            if engine != "fp32":
                r.set_engine(engine)
            assert net.resolved_engine() == ("tc" if pre == "neddf_nerf_tc" else "fp32"), engine
            fake.calls.clear()
            _run_all(net)
            assert _forward_calls(fake) == [(pre, e) for e in _ENTRIES], engine
    h = net._tc_handle.value
    assert [c[1] for c in fake.calls if c[0] == "neddf_nerf_tc_create"] == []  # "auto" reused the handle "tc" made
    assert fake.handles[h].layer_count == 3 and fake.handles[h].n_skips == 1
    # the tc handle is re-packed on a parameter change like the others, and released with them
    with torch.no_grad():
        net.layers[0].weight.add_(1.0)
        net.forward(Sampling(*samples(1, 3, 2)))
    assert fake.calls[-2][0] == "neddf_nerf_tc_set_weights" and fake.calls[-2][4] == 3 + 3
    net._release()
    assert h not in fake.handles and net._tc_handle is None


def test_auto_leaves_fp16_range_once_and_tc_raises(fake):
    """Status bit 4 of neddf_nerf_tc_status: "auto" raises EngineRangeError once and then runs the fp32 kernel; "tc"
    raises a plain FloatingPointError that names 65504; set_engine starts afresh; the fp32 engine reads no status."""
    r = _render()
    net = r.network_fine
    r.set_engine("auto")
    with torch.no_grad():
        _run_all(net)
    h = net._tc_handle.value
    fake.status = {h: 4}
    with pytest.raises(EngineRangeError) as ei:
        r.check_status()
    assert "65504" in str(ei.value) and net._range_fallback and net.resolved_engine() == "fp32"
    fake.calls.clear()
    with torch.no_grad():
        _run_all(net)
    assert _forward_calls(fake) == [("neddf_nerf", e) for e in _ENTRIES]
    r.check_status()  # nothing pending
    fake.status = {h: 4}  # out of range again although "auto" is already on fp32: an error, not another detour
    with pytest.raises(FloatingPointError) as ei:
        r.check_status()
    assert not isinstance(ei.value, EngineRangeError)
    r.set_engine("tc")
    assert not net._range_fallback and net.resolved_engine() == "tc"
    fake.status = {h: 4}
    with pytest.raises(FloatingPointError) as ei:
        r.check_status()
    assert not isinstance(ei.value, EngineRangeError) and "65504" in str(ei.value)
    r.set_engine("auto")
    assert net.resolved_engine() == "tc"
    r.set_engine("fp32")
    fake.calls.clear()
    r.check_status()
    assert fake.count("neddf_nerf_tc_status") == 1  # the handle exists: its word is still read (and is clear)
    fresh = _render()
    fresh.check_status()
    assert fake.count("neddf_nerf_tc_status") == 1  # no tc handle, nothing to read


def test_training_runs_the_fp32_kernel_under_tc(fake):
    """_NerfTrainFn's forward calls neddf_nerf_forward[_rays] under engine "tc": its backward recomputes that kernel."""
    r = _render()
    r.set_engine("tc")
    net = r.network_fine
    net.training_kernels = True
    pos, dd, var = samples(1, 4, 3)
    out = net(Sampling(pos, dd, var))
    assert out["density"].requires_grad
    d, o = torch.zeros(1, 3), torch.zeros(1, 3)
    net.forward_rays(d, o, torch.linspace(2, 6, 4).reshape(1, 4), "point", 0.0)
    assert _forward_calls(fake) == [("neddf_nerf", "_forward"), ("neddf_nerf", "_forward_rays")]
    assert fake.count("neddf_nerf_tc_create") == 0
