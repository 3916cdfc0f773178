"""Drop-in for neddf.network.NeuS (neddf/network/neus.py:12-162) on the CUDA path: same constructor, same module /
state_dict layout (``layers_sdf.N``, ``layers_col.N``, ``variance``) and ``forward(Sampling)``; the network runs in
one CUDA kernel (``csrc/neus_simt.cu`` behind ``neddf_neus_*``).

The reference takes the SDF normal with ``torch.autograd.grad`` (neus.py:133-142), so its forward only works with
autograd enabled - its own ``render_image`` (grad disabled, nerf_render.py:218) raises for this network.  Here the
normal is carried forward through the SDF trunk inside the kernel, so ``forward`` / ``render_rays`` under
``torch.no_grad()`` and ``render_image`` work.

Scope (SURVEY 8(f) item 3): inference.  There is no backward kernel for this variant: calling it with autograd
enabled on trainable parameters raises (train with the reference, load the checkpoint here).  No CPU / PyTorch
fallback."""
import ctypes as C
from typing import Dict, List, Optional

import torch
from torch import Tensor, nn

from . import _lib as L
from .network import BaseNeuralField
from .ray import Sampling


class NeuS(BaseNeuralField):
    def __init__(
        self,
        embed_pos_rank: int = 6,
        embed_dir_rank: int = 4,
        sdf_layer_count: int = 8,
        sdf_layer_width: int = 256,
        col_layer_count: int = 8,
        col_layer_width: int = 256,
        activation_type: str = "ReLU",
        init_variance: float = 0.3,
        skips: Optional[List[int]] = None,
    ) -> None:
        super().__init__()
        input_sdf_dim = embed_pos_rank * 6
        input_col_dim = 6 + embed_dir_rank * 6 + sdf_layer_width
        if skips is None:
            skips = [4]
        self.skips = [int(s) for s in skips]
        if activation_type not in ("ReLU", "tanhExp"):
            raise KeyError(activation_type)  # neus.py:70-75: the reference's dict lookup
        self.activation_type = activation_type
        self.embed_pos_rank, self.embed_dir_rank = int(embed_pos_rank), int(embed_dir_rank)
        self.sdf_layer_count, self.sdf_layer_width = int(sdf_layer_count), int(sdf_layer_width)
        self.col_layer_count, self.col_layer_width = int(col_layer_count), int(col_layer_width)
        # identical construction order and shapes to neus.py:83-99 (same parameters for the same torch seed)
        layers_sdf: List[nn.Module] = [nn.Linear(input_sdf_dim, sdf_layer_width)]
        layers_col: List[nn.Module] = []
        for layer_id in range(sdf_layer_count - 1):
            layers_sdf.append(nn.Linear(sdf_layer_width + (input_sdf_dim if layer_id in self.skips else 0), sdf_layer_width))
        layers_col.append(nn.Linear(input_col_dim, col_layer_width))
        for _ in range(col_layer_count - 1):
            layers_col.append(nn.Linear(col_layer_width, col_layer_width))
        layers_col.append(nn.Linear(col_layer_width, 3))
        self.layers_sdf = nn.ModuleList(layers_sdf)
        self.layers_col = nn.ModuleList(layers_col)
        self.variance = nn.Parameter(torch.tensor(init_variance))
        # kernel-side state
        self.engine = "fp32"  # the only engine of this variant; NeRFRender.set_engine may overwrite the attribute
        self._handle = None
        self._handle_device = None
        self._packed_key = None
        self._profile_events = None

    # ------------------------------------------------------------------ kernel plumbing --
    def _ordered_layers(self) -> List[nn.Linear]:
        return list(self.layers_sdf) + list(self.layers_col)

    def _config_struct(self) -> L.NeusConfig:
        c = L.NeusConfig()
        c.embed_pos_rank, c.embed_dir_rank = self.embed_pos_rank, self.embed_dir_rank
        c.sdf_layer_count, c.sdf_layer_width = self.sdf_layer_count, self.sdf_layer_width
        c.col_layer_count, c.col_layer_width = self.col_layer_count, self.col_layer_width
        c.activation_type = L.ACT_IDS[self.activation_type]
        if len(self.skips) > L.MAX_SKIPS:
            raise NotImplementedError("neddf_b200: more than 8 skip connections")
        c.n_skips = len(self.skips)
        for i, s in enumerate(self.skips):
            c.skips[i] = s
        return c

    def _release(self) -> None:
        if self._handle is not None:
            L.lib().neddf_neus_destroy(self._handle)
        self._handle, self._handle_device, self._packed_key = None, None, None

    def __del__(self):
        try:
            self._release()
        except Exception:  # interpreter shutdown
            pass

    def _field(self, device: torch.device):
        lib = L.lib()
        if device.type != "cuda":
            raise RuntimeError("neddf_b200.NeuS runs on CUDA devices only: move the module with .to('cuda') "
                               "(the hot path has no CPU implementation)")
        if self._handle is None or self._handle_device != device:
            self._release()
            h = C.c_void_p()
            with torch.cuda.device(device):
                cfg = self._config_struct()
                L.check(lib.neddf_neus_create(C.byref(cfg), C.byref(h)), "neus_create")
            self._handle, self._handle_device = h, device
        layers = self._ordered_layers()
        tensors = [p for l in layers for p in (l.weight, l.bias)] + [self.variance]
        key = tuple((p.data_ptr(), p._version) for p in tensors)
        if key != self._packed_key:
            for p in tensors:
                if p.dtype != torch.float32 or not p.is_contiguous() or p.device != device:
                    raise RuntimeError("neddf_b200: parameters must be contiguous fp32 tensors on the module's device")
            n = len(layers)
            ws = (C.c_void_p * n)(*[l.weight.data_ptr() for l in layers])
            bs = (C.c_void_p * n)(*[l.bias.data_ptr() for l in layers])
            with torch.cuda.device(device):
                L.check(lib.neddf_neus_set_weights(self._handle, ws, bs, n, L.ptr(self.variance), L.stream_ptr(device)),
                        "neus_set_weights")
            self._packed_key = key
        return self._handle

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self._packed_key = None  # .to()/.cuda() replaced the parameter storage
        return r

    def invalidate(self) -> None:
        self._packed_key = None

    def __getstate__(self):
        d = self.__dict__.copy()
        d["_handle"], d["_handle_device"], d["_packed_key"], d["_profile_events"] = None, None, None, None
        return d

    def check_engine_status(self) -> None:
        """(fp32 kernel: no range checks to report)"""

    def _refuse_autograd(self) -> None:
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError(
                "neddf_b200.NeuS is forward-only on the CUDA path (no backward kernel for this variant): wrap the call "
                "in torch.no_grad() / use render_image, or train with the reference and load the checkpoint")

    @staticmethod
    def _outputs(B: int, S: int, device, with_normal: bool) -> Dict[str, Tensor]:
        out = {"sdf": torch.empty(B, S, device=device, dtype=torch.float32),
               "density": torch.empty(B, S, device=device, dtype=torch.float32),
               "color": torch.empty(B, S, 3, device=device, dtype=torch.float32)}
        if with_normal:
            out["normal"] = torch.empty(B, S, 3, device=device, dtype=torch.float32)
        return out

    # ----------------------------------------------------------------------- forward --
    def forward(self, sampling: Sampling, with_normal: bool = False) -> Dict[str, Tensor]:
        """neus.py:101-162: {'sdf': [B,S], 'density': [B,S], 'color': [B,S,3]}; ``with_normal`` adds the gradient
        d sdf / d position [B,S,3] that the reference feeds to the colour trunk (neus.py:133-146) but does not return."""
        self._refuse_autograd()
        pos = L.require_cuda_f32(sampling.sample_pos, "sample_pos")
        sdir = L.require_cuda_f32(sampling.sample_dir, "sample_dir")
        B, S = pos.shape[0], pos.shape[1]
        device = pos.device
        out = self._outputs(B, S, device, with_normal)
        h = self._field(device)
        with torch.cuda.device(device):
            L.check(L.lib().neddf_neus_forward(h, L.ptr(pos), L.ptr(sdir), B * S, L.ptr(out["sdf"]), L.ptr(out["density"]),
                                               L.ptr(out["color"]), L.ptr(out.get("normal")), L.stream_ptr(device)),
                    "neus_forward")
        return out

    def forward_rays(self, ray_dir: Tensor, ray_orig: Tensor, dists: Tensor, sampling_type: str, ray_radius: float,
                     need_penalty: bool = True, need_aux: bool = True, with_normal: bool = False) -> Dict[str, Tensor]:
        """Same network with the sample geometry fused into the kernel (what NeRFRender calls; this variant has
        neither penalties nor auxiliary fields, the flags are accepted for interface parity)."""
        self._refuse_autograd()
        ray_dir = L.require_cuda_f32(ray_dir, "ray_dir")
        ray_orig = L.require_cuda_f32(ray_orig, "ray_orig")
        dists = L.require_cuda_f32(dists, "dists")
        B, S = dists.shape
        device = dists.device
        out = self._outputs(B, S, device, with_normal)
        h = self._field(device)
        prof = self._profile_events
        if prof is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(torch.cuda.current_stream(device))
        with torch.cuda.device(device):
            L.check(L.lib().neddf_neus_forward_rays(h, L.ptr(ray_dir), L.ptr(ray_orig), L.ptr(dists), B, S,
                                                    L.SAMPLING_IDS[sampling_type], float(ray_radius), L.ptr(out["sdf"]),
                                                    L.ptr(out["density"]), L.ptr(out["color"]), L.ptr(out.get("normal")),
                                                    L.stream_ptr(device)), "neus_forward_rays")
        if prof is not None:
            e1.record(torch.cuda.current_stream(device))
            prof.append((e0, e1, B * S))
        return out
