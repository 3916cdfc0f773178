"""Host plumbing shared by the field networks, over a fake library on CPU tensors: the lifecycle of every kernel handle
(create / re-pack / destroy, copies and pickles), the NeDDF training backward's gradient assembly against its fp64
statement, and FusedAdam over NeRF and NeuS renders."""
import contextlib
import copy
import ctypes as C
import pickle

import numpy as np
import pytest
import torch

import neddf_b200
from neddf_b200 import _lib as L
from neddf_b200 import optim
from neddf_b200._host import KernelHandle
from neddf_b200.network import BaseNeuralField
from neddf_b200.ray import Sampling

FP = C.POINTER(C.c_float)


class FakeLib:
    """Records every call; handles are counters, ``neddf_field_backward[_samples]`` fill their outputs with seeded values
    and ``neddf_wgrad`` / ``neddf_colsum_value_rows`` are numpy on the very pointers, strides and tiles the glue passes."""

    def __init__(self):
        self.calls, self.handles, self.next = [], {}, 100

    @staticmethod
    def arr(p, n):
        addr = p.value if hasattr(p, "value") else p
        return np.ctypeslib.as_array(C.cast(addr, FP), shape=(int(n),))

    def count(self, name):
        return sum(c[0] == name for c in self.calls)

    def __getattr__(self, name):
        if name.endswith("_create"):
            def create(cfg_ref, h_ref):
                self.next += 1
                h_ref._obj.value = self.next
                cfg = type(cfg_ref._obj)()
                C.memmove(C.byref(cfg), C.byref(cfg_ref._obj), C.sizeof(cfg))
                self.handles[self.next] = cfg
                self.calls.append((name, self.next))
                return 0
            return create
        if name.endswith("_destroy"):
            def destroy(h):
                assert self.handles.pop(h.value, None) is not None, "destroyed twice or never created"
                self.calls.append((name, h.value))
                return 0
            return destroy

        def call(*args):
            self.calls.append((name,) + args)
            return 0
        return call

    def neddf_last_error(self):
        return b"fake"

    def neddf_wgrad_workspace_bytes(self):
        return 4096

    def _fill_backward(self, h, n, bufs, seed):
        cfg = self.handles[h.value]
        n_hidden = cfg.ddf_layer_count - 1 + cfg.col_layer_count - 1
        n_e0, off_h = 6 * cfg.embed_pos_rank, 6 * (cfg.embed_pos_rank + cfg.embed_dir_rank) + 3
        sizes = [n_hidden * n * 4 * 256, n_hidden * n * 4 * 256, n * 4 * 2, n * 4 * 4, n * 4 * n_e0, n * 4 * off_h]
        rng = np.random.default_rng(seed)
        for p, size in zip(bufs, sizes):  # post, gpre, ghead_da, ghead_col, xes, xcol
            self.arr(p, size)[:] = rng.standard_normal(size).astype(np.float32)
        self.calls.append(("backward", n))
        return 0

    def neddf_field_backward(self, h, st, a, b, c, B, S, stype, radius, save, gd, gc, gp, *rest):
        return self._fill_backward(h, B * S, rest[:6], 1)

    def neddf_field_backward_samples(self, h, st, a, b, c, n, save, gd, gc, gp, *rest):
        return self._fill_backward(h, n, rest[:6], 2)

    def neddf_wgrad(self, a, lda, a_col0, ka, b, ldb, rows, out, ld_out, n_cols, ws, stream):
        assert 0 < ka <= 128 and n_cols == 256 and ld_out == 256 and ldb == 256
        A = self.arr(a, rows * lda).reshape(rows, lda).astype(np.float64)
        B = self.arr(b, rows * ldb).reshape(rows, ldb).astype(np.float64)
        O = self.arr(out, (ka - 1) * ld_out + n_cols)
        res = A[:, a_col0:a_col0 + ka].T @ B
        for m in range(ka):
            O[m * ld_out:m * ld_out + n_cols] = res[m]
        self.calls.append(("neddf_wgrad",))
        return 0

    def neddf_colsum_value_rows(self, g, n_samples, stride, out, ws, stream):
        Gm = self.arr(g, (n_samples - 1) * stride + 256)
        self.arr(out, 256)[:] = np.stack([Gm[s * stride:s * stride + 256] for s in range(n_samples)]).astype(np.float64).sum(0)
        self.calls.append(("neddf_colsum_value_rows",))
        return 0


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(L, "lib", lambda: lib)
    monkeypatch.setattr(L, "stream_ptr", lambda device=None: None)
    monkeypatch.setattr(L, "require_cuda_f32", lambda t, name: t.to(torch.float32).contiguous())
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    # CPU tensors: the forward handle's CUDA-only check is the one thing bypassed
    monkeypatch.setattr(BaseNeuralField, "_field", lambda self, device: self._HANDLES[0].get(self, device))
    seen, get = [], KernelHandle.get

    def tracked_get(kh, net, device):
        seen.append((kh, net))
        return get(kh, net, device)

    monkeypatch.setattr(KernelHandle, "get", tracked_get)
    yield lib
    for kh, net in seen:  # fake handles must never reach the real library's destroy (module __del__ after the test)
        kh.reset(net)


def small(kind):
    torch.manual_seed(0)
    if kind == "neddf":
        return neddf_b200.NeDDF(embed_pos_rank=3, embed_dir_rank=2, ddf_layer_count=4, col_layer_count=3, skips=[1])
    if kind == "nerf":
        return neddf_b200.NeRF(embed_pos_rank=3, embed_dir_rank=2, layer_count=4, skips=[1])
    return neddf_b200.NeuS(embed_pos_rank=3, embed_dir_rank=2, sdf_layer_count=3, col_layer_count=2, skips=[0])


SLOTS = [("neddf", 0), ("nerf", 0), ("nerf", 1), ("neus", 0), ("neus", 1)]


@pytest.mark.parametrize("kind,slot", SLOTS)
def test_handle_lifecycle(fake, kind, slot):
    net = small(kind)
    h = net._HANDLES[slot]
    prefix = h.prefix
    cpu = torch.device("cpu")
    sets = lambda: fake.count(prefix + "_set_weights")  # noqa: E731
    first = h.get(net, cpu)
    assert fake.count(prefix + "_create") == 1 and sets() == 1
    assert h.get(net, cpu) is first and sets() == 1  # a repeated call neither creates nor re-packs
    set_call = [c for c in fake.calls if c[0] == prefix + "_set_weights"][-1]
    n = len(net._ordered_layers())
    assert set_call[4] == n and len(set_call) == 6 + (kind == "neus")  # NeuS passes the variance pointer too
    with torch.no_grad():
        net._ordered_layers()[-1].bias.add_(1.0)  # in place: bumps the version counter
    h.get(net, cpu)
    assert sets() == 2
    net.invalidate()
    h.get(net, cpu)
    assert sets() == 3
    net.to(torch.float32)
    h.get(net, cpu)
    assert sets() == 4 and fake.count(prefix + "_create") == 1
    # a device change destroys the old handle and packs a new one
    net.to("meta")
    second = h.get(net, torch.device("meta"))
    assert [c[1] for c in fake.calls if c[0] == prefix + "_destroy"] == [first.value]
    assert fake.count(prefix + "_create") == 2 and sets() == 5 and second.value != first.value
    assert getattr(net, h.names[0]) is second and getattr(net, h.names[1]) == torch.device("meta")
    for other in net._HANDLES:
        other.get(net, torch.device("meta"))
    live = {getattr(net, o.names[0]).value for o in net._HANDLES}
    net._release()
    assert all(getattr(net, name) is None for o in net._HANDLES for name in o.names)
    assert not live & set(fake.handles)  # every handle destroyed


@pytest.mark.parametrize("kind,slot,bad", [(k, s, b) for k, s in SLOTS for b in ("float64 bias", "strided bias")] +
                         [("neus", s, "float64 variance") for s in (0, 1)])
def test_bad_parameters_are_refused_before_any_repack(fake, kind, slot, bad):
    net = small(kind)
    h = net._HANDLES[slot]
    bias = net._ordered_layers()[1].bias
    if bad == "float64 bias":
        bias.data = bias.data.double()
    elif bad == "strided bias":
        bias.data = torch.zeros(2 * bias.shape[0])[::2]
    else:
        net.variance.data = net.variance.data.double()
    with pytest.raises(RuntimeError, match="contiguous fp32"):
        h.get(net, torch.device("cpu"))
    assert fake.count(h.prefix + "_set_weights") == 0
    net._release()


def _neddf_expected(net, post, gpre, gda, gcol, xes, xcol):
    """fp64 statement of every NeDDF parameter gradient from what the backward left: [parts]^T gpre_l per layer (skip
    layers: [xes | post], colour layer 0: [xcol | post]), bias = sum of the value rows, and the heads."""
    n_ddf, n_col = net.ddf_layer_count - 1, net.col_layer_count - 1
    R = post.shape[1] * 4
    rows = lambda t: t.reshape(R, -1)  # noqa: E731
    exp = []
    for l in range(n_ddf + n_col):
        if l == 0:
            parts = [xes]
        elif l < n_ddf:
            parts = ([xes] if (l - 1) in net.skips else []) + [post[l - 1]]
        elif l == n_ddf:
            parts = [xcol, post[n_ddf - 1]]
        else:
            parts = [post[l - 1]]
        X = np.concatenate([rows(p) for p in parts], 1)
        exp += [X.T @ rows(gpre[l]), gpre[l][:, 0, :].sum(0)]
    gda_t = rows(gda).T @ rows(post[n_ddf - 1])
    exp += [gda_t[0][:, None], gda[:, 0, 0:1].sum(0), gda_t[1][:, None], gda[:, 0, 1:2].sum(0)]
    exp += [(rows(gcol)[:, :3].T @ rows(post[-1])).T, gcol[:, 0, :3].sum(0)]
    return exp


@pytest.mark.parametrize("path", ["rays", "samples"])
def test_neddf_training_backward_assembles_every_gradient(fake, path):
    net = small("neddf")
    B, S = 3, 5
    n = B * S
    g = torch.Generator().manual_seed(3)
    captured = {}
    orig = fake._fill_backward

    def fill(h, n_, bufs, seed):  # keep what the fake kernel wrote, as fp64
        rc = orig(h, n_, bufs, seed)
        n_hidden = net.ddf_layer_count - 1 + net.col_layer_count - 1
        shapes = [(n_hidden, n, 4, 256), (n_hidden, n, 4, 256), (n, 4, 2), (n, 4, 4), (n, 4, 18), (n, 4, 33)]
        captured["bufs"] = [fake.arr(p, np.prod(s)).reshape(s).astype(np.float64) for p, s in zip(bufs, shapes)]
        return rc

    fake._fill_backward = fill
    if path == "rays":
        d, o = torch.randn(B, 3, generator=g), torch.randn(B, 3, generator=g)
        dists = torch.sort(torch.rand(B, S, generator=g), 1)[0] + 1
        out = net.forward_rays(d, o, dists, "cone", 0.01)
    else:
        out = net.forward(Sampling(*(torch.randn(B, S, 3, generator=g) for _ in range(3))))
    loss = sum((out[k] * torch.randn(out[k].shape, generator=g)).sum() for k in ("density", "color", "fields_penalty"))
    loss.backward()
    assert fake.count("backward") == 1
    exp = _neddf_expected(net, *captured["bufs"])
    params = net._param_tensors()
    assert len(params) == len(exp)
    for i, (p, e) in enumerate(zip(params, exp)):
        assert p.grad is not None and tuple(p.grad.shape) == e.shape, (i, p.grad, e.shape)
        np.testing.assert_allclose(p.grad.numpy(), e, rtol=2e-5, atol=2e-5 * np.abs(e).max(), err_msg=str(i))
    # a NeDDF that has run a backward holds a workspace: copies and pickles carry none of its kernel-side state
    assert isinstance(net._wgrad_ws, torch.Tensor)
    net._profile_events = []
    for twin in (copy.deepcopy(net), pickle.loads(pickle.dumps(net))):
        assert not hasattr(twin, "_wgrad_ws") and twin._profile_events is None
        assert twin._handle is None and twin._handle_device is None and twin._packed_key is None
        assert all(torch.equal(a, b) for a, b in zip(net.state_dict().values(), twin.state_dict().values()))
    assert net._handle is not None and net._packed_key is not None and net._profile_events == []
    net._release()


@pytest.mark.parametrize("target", ["neddf.network.NeRF", "neddf.network.NeuS"])
def test_fused_adam_steps_nerf_and_neus_without_a_field_handle(fake, target):
    r = neddf_b200.NeRFRender(network_config={"_target_": target, "embed_pos_rank": 3, "embed_dir_rank": 2, "skips": [1]},
                              use_coarse_network=True)
    nets = {id(n): n for n in (r.network_coarse, r.network_fine)}.values()
    s = Sampling(*(torch.randn(1, 4, 3) for _ in range(3)))
    prefix = r.network_fine._HANDLES[0].prefix
    with torch.no_grad():
        for net in nets:
            net.forward(s)
            net.forward(s)
    assert fake.count(prefix + "_set_weights") == len(nets)  # one pack per network, none on the repeated call
    for p in r.get_parameters_list():
        p.grad = torch.ones_like(p)
    optim.FusedAdam.for_render(r, lr=1e-3).step()
    steps = [c for c in fake.calls if c[0] == "neddf_field_adam_step"]
    assert steps and all(c[1] is None for c in steps)  # only a NeDDF handle is a neddf_field_t*
    with torch.no_grad():
        for net in nets:
            net.forward(s)
            net.forward(s)
    assert fake.count(prefix + "_set_weights") == 2 * len(nets)  # the next forward re-packs exactly once
    for net in nets:
        net._release()
