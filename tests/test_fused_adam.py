"""FusedAdam's host logic over a fake library, on CPU tensors: the fake ``neddf_field_adam_step`` applies adam_kernel's
fp32 arithmetic (csrc/train_glue.cu) to the very pointers it is given and records every call, and each test runs
FusedAdam and ``torch.optim.Adam(foreach=False)`` side by side on identical parameters and gradients.  After every step
the parameters and the ``exp_avg`` / ``exp_avg_sq`` states agree to 1e-6 and the per-parameter step counts are equal:
over NeDDF, NeRF and NeuS renders, several parameter groups, an lr scheduler, zero and missing gradients, groups added
later, the 64-tensor slicing of a call, state dicts moved between the two optimisers and ``step(closure)``."""
import contextlib

import numpy as np
import pytest
import torch

import neddf_b200
from neddf_b200 import _lib as L
from neddf_b200 import optim
from neddf_b200._host import KernelHandle
from neddf_b200.network import BaseNeuralField
from tests.test_field_host_glue import FakeLib

TOL = 1e-6
NET_CFG = {
    "neddf": {"_target_": "neddf.network.NeDDF", "embed_pos_rank": 3, "embed_dir_rank": 2, "ddf_layer_count": 4,
              "col_layer_count": 3, "skips": [1]},
    "nerf": {"_target_": "neddf.network.NeRF", "embed_pos_rank": 3, "embed_dir_rank": 2, "layer_count": 4, "skips": [1]},
    "neus": {"_target_": "neddf.network.NeuS", "embed_pos_rank": 3, "embed_dir_rank": 2, "sdf_layer_count": 3,
             "col_layer_count": 2, "skips": [0]},
}


def _r32(x):
    """Round to fp32 (one kernel operation), kept as fp64 for the next one."""
    return np.asarray(x, dtype=np.float64).astype(np.float32).astype(np.float64)


class AdamLib(FakeLib):
    """FakeLib whose ``neddf_field_adam_step`` refuses what the C function refuses and otherwise runs adam_kernel's
    arithmetic in numpy (fp32 rounding after every operation) on the passed pointers; ``adam`` records
    (handle, n_tensors, lr, betas, eps, weight_decay, step) per call."""

    def __init__(self):
        super().__init__()
        self.adam = []

    def neddf_field_adam_step(self, f, P, G, M, V, N, n, lr, b1, b2, eps, wd, step, stream):
        h = None if f is None else (f.value if hasattr(f, "value") else f)
        assert 1 <= n <= 64 and step >= 1, (n, step)
        assert all(P[i] and G[i] and M[i] and V[i] and N[i] >= 0 for i in range(n))
        if h is not None:
            cfg = self.handles[h]
            assert n == 2 * (cfg.ddf_layer_count - 1 + cfg.col_layer_count - 1 + 3), n
        self.adam.append((h, n, lr, (b1, b2), eps, wd, step))
        bc1 = _r32(1.0 - b1 ** step)  # betas arrive as doubles; lr, eps and weight_decay as fp32
        bc2_sqrt = _r32(np.sqrt(1.0 - b2 ** step))
        omb1, omb2 = _r32(1.0 - b1), _r32(1.0 - b2)
        lr, b1, b2, eps, wd = (float(np.float32(x)) for x in (lr, b1, b2, eps, wd))
        size = _r32(lr / bc1)
        for i in range(n):
            p, g, m, v = (self.arr(a[i], N[i]) for a in (P, G, M, V))
            gi = g.astype(np.float64)
            if wd != 0.0:
                gi = _r32(wd * p + gi)
            d = _r32(gi - m)  # exp_avg.lerp_(g, 1 - b1)
            mi = _r32(m + omb1 * d) if omb1 < 0.5 else _r32(gi - _r32(d * _r32(1.0 - omb1)))
            vi = _r32(b2 * v + _r32(_r32(omb2 * gi) * gi))
            den = _r32(_r32(_r32(np.sqrt(vi)) / bc2_sqrt) + eps)
            p[:] = _r32(p - _r32(size * _r32(mi / den)))
            m[:], v[:] = mi, vi
        return 0


@pytest.fixture
def fake(monkeypatch):
    lib = AdamLib()
    monkeypatch.setattr(L, "lib", lambda: lib)
    monkeypatch.setattr(L, "stream_ptr", lambda device=None: None)
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


def _render(kind, twin_of=None):
    torch.manual_seed(0)
    r = neddf_b200.NeRFRender(network_config=dict(NET_CFG[kind]), use_coarse_network=True)
    if twin_of is not None:
        r.load_state_dict(twin_of.state_dict())
    return r


def _renders(kind):
    a = _render(kind)
    return a, _render(kind, a)


def _plain(n, seed=5):
    """``n`` parameter tensors outside any network, of mixed sizes, and their twins."""
    g = torch.Generator().manual_seed(seed)
    ps = [torch.randn(int(s), generator=g) for s in torch.randint(1, 40, (n,), generator=g)]
    return [p.clone().requires_grad_(True) for p in ps], [p.clone().requires_grad_(True) for p in ps]


def _torch_adam(params, **kw):
    return torch.optim.Adam(params, foreach=False, **kw)


def _set_grads(fused_params, ref_params, gen, skip=()):
    """The same random gradient on both twins (magnitudes spread over four decades); None for ``skip`` indices."""
    for i, (a, b) in enumerate(zip(fused_params, ref_params)):
        if i in skip:
            a.grad = b.grad = None
            continue
        g = torch.randn(a.shape, generator=gen) * 10.0 ** torch.empty(a.shape).uniform_(-3, 1, generator=gen)
        a.grad, b.grad = g.clone(), g.clone()


def _close(a, b, what, terms=None):
    """|a - b| <= TOL (|b| + max|b| + |terms|): relative to the element and its tensor, and, where the update may cancel
    (exp_avg = b1 m + (1 - b1) g near 0), to the size of the terms it sums."""
    a, b = a.detach().double().numpy(), b.detach().double().numpy()
    scale = float(np.abs(b).max()) if b.size else 0.0
    if terms is not None:
        scale = scale + np.abs(terms.detach().double().numpy())
    bad = np.abs(a - b) > TOL * (np.abs(b) + scale)
    assert not bad.any(), (what, float(np.abs(a - b).max()), scale)


def _compare(fo, ro, fused_params, ref_params, what="", before=None):
    """Parameters, moments and step counts of FusedAdam ``fo`` against torch.optim.Adam ``ro``; ``before``: the
    reference parameters before the step (a parameter near 0 may be the difference of two larger terms)."""
    for i, (a, b) in enumerate(zip(fused_params, ref_params)):
        _close(a, b, (what, i, "param"), None if before is None else before[i])
        sa, sb = fo.state.get(a, {}), ro.state.get(b, {})
        assert bool(sa) == bool(sb), (what, i)
        if sb:
            assert float(sa["step"]) == float(sb["step"]), (what, i, float(sa["step"]), float(sb["step"]))
            assert sa["step"].dtype == torch.float32 and sa["step"].device.type == "cpu"
            _close(sa["exp_avg"], sb["exp_avg"], (what, i, "exp_avg"), b.grad)
            _close(sa["exp_avg_sq"], sb["exp_avg_sq"], (what, i, "exp_avg_sq"))


def _step(fo, ro, fused_params, ref_params, what=""):
    """One step of both optimisers, then ``_compare``."""
    before = [p.detach().clone() for p in ref_params]
    fo.step()
    ro.step()
    _compare(fo, ro, fused_params, ref_params, what, before)


def _nets(r):
    return list({id(n): n for n in (r.network_coarse, r.network_fine)}.values())


@pytest.mark.parametrize("kind", ["neddf", "nerf", "neus"])
def test_for_render_matches_torch_adam(fake, kind):
    """One group over a render's coarse and fine networks, 5 steps.  A NeDDF is stepped through its handle, one call
    per network; a NeRF or NeuS has none - one call per network, NeuS's two variances in one more - and is
    invalidated so that its next call re-packs."""
    rf, rr = _renders(kind)
    pf, pr = rf.get_parameters_list(), rr.get_parameters_list()
    fo, ro = optim.FusedAdam.for_render(rf, lr=1e-2), _torch_adam(pr, lr=1e-2)
    gen = torch.Generator().manual_seed(1)
    for it in range(5):
        _set_grads(pf, pr, gen)
        fake.adam.clear()
        _step(fo, ro, pf, pr, it)
        handles = [c[0] for c in fake.adam]
        if kind == "neddf":
            assert len(handles) == 2 and all(h is not None for h in handles)
            assert all(net._packed_key is not None for net in _nets(rf))  # re-packed by the step itself
        else:
            assert handles == [None] * (3 if kind == "neus" else 2)
            assert all(net._packed_key is None for net in _nets(rf))
        assert {c[6] for c in fake.adam} == {it + 1}


def test_two_param_groups_keep_their_hyperparameters(fake):
    """Coarse and fine NeDDF networks in two groups with different lr, betas, eps and weight_decay: each network still
    goes through its handle, with its own group's values."""
    rf, rr = _renders("neddf")
    hyper = [dict(lr=2e-2, betas=(0.8, 0.99), eps=1e-6, weight_decay=0.0),
             dict(lr=5e-3, betas=(0.5, 0.9), eps=1e-3, weight_decay=1e-2)]
    fo = optim.FusedAdam([dict(params=list(rf.network_coarse.parameters()), **hyper[0]),
                          dict(params=list(rf.network_fine.parameters()), **hyper[1])], networks=_nets(rf))
    ro = _torch_adam([dict(params=list(rr.network_coarse.parameters()), **hyper[0]),
                      dict(params=list(rr.network_fine.parameters()), **hyper[1])])
    pf, pr = rf.get_parameters_list(), rr.get_parameters_list()
    gen = torch.Generator().manual_seed(2)
    for it in range(5):
        _set_grads(pf, pr, gen)
        fake.adam.clear()
        _step(fo, ro, pf, pr, it)
        assert len(fake.adam) == 2 and all(c[0] is not None for c in fake.adam)
        for c, h in zip(fake.adam, hyper):
            assert (c[2], c[3], c[4], c[5]) == (h["lr"], h["betas"], h["eps"], h["weight_decay"])


def test_network_split_across_groups_is_stepped_without_its_handle(fake):
    """The coarse NeDDF's tensors sit in two groups, so it cannot be stepped in one handle call: its part of each group
    goes through the no-handle path and the network is invalidated.  The fine network, whole in the second group,
    still goes through its handle."""
    rf, rr = _renders("neddf")
    pf, pr = rf.get_parameters_list(), rr.get_parameters_list()
    fo = optim.FusedAdam([dict(params=pf[:6]), dict(params=pf[6:], lr=3e-3)], lr=1e-2, networks=_nets(rf))
    ro = _torch_adam([dict(params=pr[:6]), dict(params=pr[6:], lr=3e-3)], lr=1e-2)
    gen = torch.Generator().manual_seed(3)
    for it in range(5):
        _set_grads(pf, pr, gen)
        fake.adam.clear()
        _step(fo, ro, pf, pr, it)
        assert [c[0] is not None for c in fake.adam] == [False, True, False]
        assert rf.network_coarse._packed_key is None and rf.network_fine._packed_key is not None


@pytest.mark.parametrize("kind", ["neddf", "nerf"])
def test_exponential_lr_between_steps(fake, kind):
    """ExponentialLR stepped after every optimiser step (nerf_trainer.py:43,64): each call carries the decayed lr."""
    rf, rr = _renders(kind)
    pf, pr = rf.get_parameters_list(), rr.get_parameters_list()
    fo, ro = optim.FusedAdam.for_render(rf, lr=1e-2), _torch_adam(pr, lr=1e-2)
    sf, sr = torch.optim.lr_scheduler.ExponentialLR(fo, 0.5), torch.optim.lr_scheduler.ExponentialLR(ro, 0.5)
    gen = torch.Generator().manual_seed(4)
    for it in range(5):
        _set_grads(pf, pr, gen)
        fake.adam.clear()
        _step(fo, ro, pf, pr, it)
        sf.step()
        sr.step()
        assert {c[2] for c in fake.adam} == {1e-2 * 0.5 ** it}


def test_zero_grads_still_step(fake):
    """zero_grad(set_to_none=False) leaves zero gradients, not None: those parameters are stepped (their moments decay,
    their step counts advance) exactly as torch does."""
    rf, rr = _renders("neddf")
    pf, pr = rf.get_parameters_list(), rr.get_parameters_list()
    fo, ro = optim.FusedAdam.for_render(rf, lr=1e-2), _torch_adam(pr, lr=1e-2)
    gen = torch.Generator().manual_seed(5)
    _set_grads(pf, pr, gen)
    fo.step()
    ro.step()
    for it in range(4):
        fo.zero_grad(set_to_none=False)
        ro.zero_grad(set_to_none=False)
        for i in range(it % 2, len(pf), 2):  # every other tensor gets a gradient, the rest keep zeros
            g = torch.randn(pf[i].shape, generator=gen)
            pf[i].grad.add_(g)
            pr[i].grad.add_(g)
        fake.adam.clear()
        _step(fo, ro, pf, pr, it)
        assert len(fake.adam) == 2 and all(c[0] is not None for c in fake.adam)


def test_late_gradient_uses_its_own_step_count(fake):
    """A tensor (and, in the fine network, a whole layer) without a gradient on the first two steps: torch skips it
    and starts its step count at its first gradient, so its bias corrections are those of step 1, 2, 3 while the
    others are at 3, 4, 5.  Mixed step counts in a network mean no handle call, one call per step count, and a
    re-pack on the next use."""
    rf, rr = _renders("neddf")
    pf, pr = rf.get_parameters_list(), rr.get_parameters_list()
    fo, ro = optim.FusedAdam.for_render(rf, lr=1e-2), _torch_adam(pr, lr=1e-2)
    n_coarse = len(list(rf.network_coarse.parameters()))
    late = {1, n_coarse + 2, n_coarse + 3}
    gen = torch.Generator().manual_seed(6)
    for it in range(5):
        _set_grads(pf, pr, gen, skip=late if it < 2 else ())
        fake.adam.clear()
        _step(fo, ro, pf, pr, it)
        if it < 2:
            assert [c[6] for c in fake.adam] == [it + 1]  # both networks, one no-handle call
        else:
            assert sorted(c[6] for c in fake.adam) == [it - 1, it + 1]
        assert all(c[0] is None for c in fake.adam)
        assert all(net._packed_key is None for net in _nets(rf))


def test_add_param_group_later(fake):
    """The fine network joins as a second group after two steps: its step counts start at 1, and as all its tensors
    share one count it goes through its handle."""
    rf, rr = _renders("neddf")
    fo = optim.FusedAdam(rf.network_coarse.parameters(), lr=1e-2, networks=_nets(rf))
    ro = _torch_adam(rr.network_coarse.parameters(), lr=1e-2)
    pf, pr = rf.get_parameters_list(), rr.get_parameters_list()
    n_coarse = len(list(rf.network_coarse.parameters()))
    gen = torch.Generator().manual_seed(7)
    for it in range(5):
        if it == 2:
            fo.add_param_group(dict(params=list(rf.network_fine.parameters()), lr=4e-3, weight_decay=1e-2))
            ro.add_param_group(dict(params=list(rr.network_fine.parameters()), lr=4e-3, weight_decay=1e-2))
        _set_grads(pf, pr, gen, skip=range(n_coarse, len(pf)) if it < 2 else ())
        fake.adam.clear()
        _step(fo, ro, pf, pr, it)
        assert [(c[0] is not None, c[6]) for c in fake.adam] == [(True, it + 1)] + ([(True, it - 1)] if it >= 2 else [])


def test_more_than_64_tensors_are_sliced(fake):
    """150 tensors outside any network go in calls of at most 64 tensors."""
    pf, pr = _plain(150)
    fo, ro = optim.FusedAdam(pf, lr=1e-2, weight_decay=1e-2), _torch_adam(pr, lr=1e-2, weight_decay=1e-2)
    gen = torch.Generator().manual_seed(8)
    for it in range(5):
        _set_grads(pf, pr, gen)
        fake.adam.clear()
        _step(fo, ro, pf, pr, it)
        assert [c[1] for c in fake.adam] == [64, 64, 22] and all(c[0] is None for c in fake.adam)


def _resume(first, second):
    """2 steps with optimiser ``first``, its state dict loaded into a fresh ``second`` on a copy of the parameters, 3
    more steps; against torch.optim.Adam run uninterrupted for all 5."""
    r0, r1 = _renders("neddf")
    r2 = _render("neddf", r0)
    make = {"fused": lambda r, **kw: optim.FusedAdam.for_render(r, **kw),
            "torch": lambda r, **kw: _torch_adam(r.get_parameters_list(), **kw)}
    kw = dict(lr=1e-2, weight_decay=1e-3)
    ref = _torch_adam(r0.get_parameters_list(), **kw)
    o1 = make[first](r1, **kw)
    p0, p1 = r0.get_parameters_list(), r1.get_parameters_list()
    gen = torch.Generator().manual_seed(9)
    for it in range(2):
        _set_grads(p1, p0, gen)
        o1.step()
        ref.step()
    r2.load_state_dict(r1.state_dict())
    o2 = make[second](r2, lr=0.5)  # the state dict brings the group's lr back
    o2.load_state_dict(o1.state_dict())
    p2 = r2.get_parameters_list()
    for it in range(3):
        _set_grads(p2, p0, gen)
        if second == "fused":
            _step(o2, ref, p2, p0, it)
        else:  # the roles swap: the uninterrupted run is the one with FusedAdam's state layout
            _step(ref, o2, p0, p2, it)


@pytest.mark.parametrize("first,second", [("fused", "fused"), ("fused", "torch"), ("torch", "fused")])
def test_state_dict_round_trip(fake, first, second):
    _resume(first, second)


def test_step_with_closure(fake):
    """step(closure): the closure runs with autograd enabled (it calls backward) and its loss is returned."""
    pf, pr = _plain(20)
    fo, ro = optim.FusedAdam(pf, lr=1e-2), _torch_adam(pr, lr=1e-2)
    gen = torch.Generator().manual_seed(10)
    for it in range(5):
        w = [torch.randn(p.shape, generator=gen) for p in pf]

        def closure(opt, ps):
            opt.zero_grad()
            loss = sum((torch.sin(p) * c).sum() for p, c in zip(ps, w))
            loss.backward()
            return loss

        before = [p.detach().clone() for p in pr]
        lf = fo.step(lambda: closure(fo, pf))
        lr = ro.step(lambda: closure(ro, pr))
        assert abs(float(lf.detach()) - float(lr.detach())) <= 1e-5 * abs(float(lr.detach()))
        _compare(fo, ro, pf, pr, it, before)
