"""Adam with the kernel-layout weight re-pack fused behind it (SURVEY 8(f) item 1).

The reference steps ``torch.optim.Adam`` over ``neural_render.get_parameters_list()`` (nerf_trainer.py:38-42,
129); the CUDA field kernels then need their packed copies of the weights refreshed.  ``FusedAdam`` does the
update of every tensor of a network in ONE call (``neddf_field_adam_step``, a launch per 32 tensors) and, for a
NeDDF, re-packs on the same stream, so a training step has no per-tensor optimiser kernels and no separate
"parameters changed" detection.  It is a ``torch.optim.Optimizer`` (param_groups, lr schedulers work) and keeps torch.optim.Adam's per-parameter
state (``step`` as a float32 CPU scalar tensor, ``exp_avg``, ``exp_avg_sq``), so state dicts interchange with
torch's in both directions; parameters that do not belong to one of its networks are stepped by the same kernel
without a re-pack.
"""
import ctypes as C
from typing import Dict, Iterable, List

import torch

from . import _lib as L
from .network import NeDDF

MAX_TENSORS = 64  # per neddf_field_adam_step call


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params: Iterable, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, networks: Iterable = ()) -> None:
        """``networks``: the neddf_b200 field networks whose parameters are in ``params``.  A NeDDF's packed weights
        are refreshed by the step itself; a NeRF or NeuS re-packs on its next call.  ``FusedAdam.for_render(render,
        ...)`` fills both."""
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self._networks: List = list({id(n): n for n in networks}.values())

    @classmethod
    def for_render(cls, render, **kw) -> "FusedAdam":
        nets = [render.network_coarse, render.network_fine]
        return cls(render.get_parameters_list(), networks=nets, **kw)

    def _state(self, p):
        st = self.state[p]
        if not st:  # torch.optim.Adam's layout (a state dict loaded from either optimiser has it already)
            st["step"] = torch.tensor(0.0, dtype=torch.float32)
            st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        return st

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        lib = L.lib()
        done, repacked = set(), set()
        for group in self.param_groups:
            if group.get("amsgrad") or group.get("maximize"):
                raise NotImplementedError("FusedAdam: amsgrad / maximize (from a loaded torch.optim.Adam state dict)")
            lr, (b1, b2), eps, wd = group["lr"], group["betas"], group["eps"], group["weight_decay"]
            # as torch.optim.Adam: a parameter without a gradient is skipped and its own step count stays
            live = [p for p in group["params"] if p.grad is not None]
            steps: Dict[int, int] = {}
            for p in live:
                st = self._state(p)
                st["step"] += 1
                steps[id(p)] = int(st["step"].item())
            batches = []
            for net in self._networks:
                ps = [t for l in net._ordered_layers() for t in (l.weight, l.bias)]
                if all(id(p) in steps and id(p) not in done for p in ps) and len({steps[id(p)] for p in ps}) == 1:
                    batches.append((net, ps))
                    done.update(id(p) for p in ps)
            # the rest, one batch per step count (the bias corrections are per launch)
            by_step: Dict[int, List] = {}
            for p in live:
                if id(p) not in done:
                    by_step.setdefault(steps[id(p)], []).append(p)
                    done.add(id(p))
            batches += [(None, ps) for ps in by_step.values()]
            for net, ps in batches:
                device = ps[0].device
                n = len(ps)
                grads = [p.grad.contiguous() for p in ps]
                st = [self.state[p] for p in ps]
                # the step re-packs a neddf_field_t* behind the update: only a NeDDF has one.  Without a handle the
                # launch takes at most 64 tensors.
                handle = net._field(device) if isinstance(net, NeDDF) else None
                slices = [slice(0, n)] if handle is not None else [slice(i, i + MAX_TENSORS) for i in range(0, n, MAX_TENSORS)]
                with torch.cuda.device(device):
                    for sl in slices:
                        m = len(ps[sl])
                        L.check(lib.neddf_field_adam_step(
                            handle, (C.c_void_p * m)(*[t.data_ptr() for t in ps[sl]]),
                            (C.c_void_p * m)(*[t.data_ptr() for t in grads[sl]]),
                            (C.c_void_p * m)(*[s["exp_avg"].data_ptr() for s in st[sl]]),
                            (C.c_void_p * m)(*[s["exp_avg_sq"].data_ptr() for s in st[sl]]),
                            (C.c_int64 * m)(*[p.numel() for p in ps[sl]]), m, float(lr), float(b1), float(b2), float(eps),
                            float(wd), steps[id(ps[0])], L.stream_ptr(device)), "adam_step")
                if handle is not None:
                    repacked.add(id(net))
        for net in self._networks:  # the kernel wrote parameters without bumping their version counters
            if id(net) not in repacked:
                net.invalidate()
        return loss
