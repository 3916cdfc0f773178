"""Drop-in for neddf.network.NeuS (neddf/network/neus.py:12-162) on the CUDA path: same constructor, same module /
state_dict layout (``layers_sdf.N``, ``layers_col.N``, ``variance``) and ``forward(Sampling)``; the network runs in
one CUDA kernel (``csrc/neus_simt.cu`` behind ``neddf_neus_*``).

The reference takes the SDF normal with ``torch.autograd.grad`` (neus.py:133-142), so its forward only works with
autograd enabled - its own ``render_image`` (grad disabled, nerf_render.py:218) raises for this network.  Here the
normal is carried forward through the SDF trunk inside the kernel, so ``forward`` / ``render_rays`` under
``torch.no_grad()`` and ``render_image`` work.

Scope (SURVEY 8(f) item 3): inference.  By default a call with autograd enabled on trainable parameters raises.
No CPU / PyTorch fallback.

Training (opt-in: ``net.training_kernels = True`` or NEDDF_NEUS_TRAIN=1): the backward of the autograd graph of
neus.py:101-162 with respect to the parameters - second order through the normal, which the reference takes with
autograd.grad(create_graph=True) - runs in ``csrc/neus_train.cu`` (forward recomputed per tile, data gradients in fp32
FMA) + ``neddf_wgrad`` / ``neddf_colsum_value_rows`` (weight / bias gradients).  ``forward`` / ``forward_rays`` then
return tensors with a ``grad_fn`` and ``NeRFRender.render_rays`` trains through the compositing backward."""
import ctypes as C
import os
from typing import Dict, List, Optional

import torch
from torch import Tensor, nn

from . import _lib as L
from ._host import KernelHandle, WeightGrad
from .network import BaseNeuralField
from .ray import Sampling


def unit_normals(g: Tensor) -> Tensor:
    """The SDF gradient [m,3] as unit normals (``F.normalize``: a zero gradient stays 0)."""
    return torch.nn.functional.normalize(g, dim=1)


class _NeusTrainFn(torch.autograd.Function):
    """NeuS.forward under autograd.  forward: the inference kernel (neddf_neus_forward[_rays]); backward:
    neddf_neus_train_backward[_rays] (recomputes the forward per tile, leaves the layer inputs and pre-activation
    gradients in global memory), then gW = X^T G as tensor-core split-K GEMMs (neddf_wgrad), bias gradients as column
    sums of the value rows and d variance as the sum of the per-sample terms.  Gradients flow to the module's parameters
    only (nerf_trainer.py:38-42 optimises nothing else)."""

    @staticmethod
    def forward(ctx, net, a, b, c, sampling_type, ray_radius, with_normal, *params):
        """(a, b, c) = (ray_dir[B,3], ray_orig[B,3], dists[B,S]) with a sampling type, or (pos, dir)[B,S,3] and c = None
        when sampling_type is None."""
        with torch.no_grad():
            out = net._launch_forward(a, b, c, sampling_type, ray_radius, with_normal)
        ctx.net, ctx.meta = net, (sampling_type, float(ray_radius))
        ctx.save_for_backward(a, b, c)
        return (out["sdf"], out["density"], out["color"]) + ((out["normal"],) if with_normal else ())

    @staticmethod
    def backward(ctx, g_sdf, g_density, g_color, g_normal=None):
        net = ctx.net
        a, b, c = ctx.saved_tensors
        sampling_type, ray_radius = ctx.meta
        from_rays = sampling_type is not None
        B, S = (c.shape if from_rays else a.shape[:2])
        n = B * S
        device = a.device
        W, Ls, Lc = 256, net.sdf_layer_count, net.col_layer_count
        n_e, n_x = 6 * net.embed_pos_rank, 6 + 6 * net.embed_dir_rank

        def prep(g, shape, zero_fill):
            if g is None:
                return torch.zeros(shape, device=device, dtype=torch.float32) if zero_fill else None
            return g.contiguous().to(torch.float32)

        g_sdf, g_density = prep(g_sdf, (B, S), False), prep(g_density, (B, S), True)
        g_color, g_normal = prep(g_color, (B, S, 3), True), prep(g_normal, (B, S, 3), False)
        f32 = dict(device=device, dtype=torch.float32)
        E4 = torch.empty(n, 4, n_e, **f32)
        XS = torch.empty(max(Ls - 1, 1), n, 4, W, **f32)
        GS = torch.empty(Ls, n, 4, W, **f32)
        XC0 = torch.empty(n, n_x, **f32)
        FO = torch.empty(n, W, **f32)
        XC = torch.empty(Lc, n, W, **f32)
        GC = torch.empty(Lc, n, W, **f32)
        GH = torch.empty(n, 3, **f32)
        GV = torch.empty(n, **f32)
        bufs = (C.c_void_p * 9)(*[t.data_ptr() for t in (E4, XS, GS, XC0, FO, XC, GC, GH, GV)])
        lib = L.lib()
        h = net._train_field(device)
        stream = L.stream_ptr(device)
        with torch.cuda.device(device):
            if from_rays:
                L.check(lib.neddf_neus_train_backward_rays(
                    h, L.ptr(a), L.ptr(b), L.ptr(c), B, S, L.SAMPLING_IDS[sampling_type], ray_radius, L.ptr(g_sdf),
                    L.ptr(g_density), L.ptr(g_color), L.ptr(g_normal), bufs, stream), "neus_train_backward_rays")
            else:
                L.check(lib.neddf_neus_train_backward(
                    h, L.ptr(a), L.ptr(b), n, L.ptr(g_sdf), L.ptr(g_density), L.ptr(g_color), L.ptr(g_normal), bufs, stream),
                    "neus_train_backward")
            wg = WeightGrad(net, device, n)

            def layer_grad(parts, Gm, rows, stride):
                """d weight [out, in] and d bias of a layer with inputs `parts` (A, columns) over `rows` rows."""
                gWt, gb = wg.layer(parts, Gm, rows, stride)
                return [gWt.t().contiguous(), gb]

            grads = []
            for l in range(Ls):  # layers_sdf.l over the 4 rows of every sample: in_0 = E4, in_l = [XS_{l-1} | E4 if skip]
                parts = [(E4, n_e)] if l == 0 else ([(XS[l - 1], W)] + ([(E4, n_e)] if (l - 1) in net.skips else []))
                grads += layer_grad(parts, GS[l], 4 * n, 4 * W)
            grads += layer_grad([(XC0, n_x), (FO, W)], GC[0], n, W)  # layers_col.0: [pos | dir PE | normal | F]
            for l in range(1, Lc):
                grads += layer_grad([(XC[l - 1], W)], GC[l], n, W)
            gh = wg.empty(3, W)  # the 3-channel output layer: GH^T h_{Lc-1}, already [out, in]
            wg.into(gh, 0, GH, 3, 3, XC[Lc - 1], n)
            grads += [gh, GH.sum(0), GV.sum()]
        return (None,) * 7 + tuple(grads)


class NeuS(BaseNeuralField):
    # sdf grows outward; density is a bump around the surface, not monotone across it, so it has no outside
    _MESH_VIEW_SIGN = {"sdf": -1.0}
    _TRACE_FIELD = "sdf"
    _HANDLES = (KernelHandle("neddf_neus"), KernelHandle("neddf_neus_train", "_train"))
    _GRAD_REFUSAL = (
        "neddf_b200.NeuS is forward-only on the CUDA path by default: wrap the call in torch.no_grad() / use "
        "render_image, or opt in to the training backward kernel (csrc/neus_train.cu) with "
        "net.training_kernels = True or NEDDF_NEUS_TRAIN=1")

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
        # training backward (csrc/neus_train.cu): opt-in, the default stays the forward-only refusal
        self.training_kernels = os.environ.get("NEDDF_NEUS_TRAIN", "0") not in ("", "0")

    # ------------------------------------------------------------------ kernel plumbing --
    def _ordered_layers(self) -> List[nn.Linear]:
        return list(self.layers_sdf) + list(self.layers_col)

    def _config_struct(self) -> L.NeusConfig:
        c = L.NeusConfig()
        c.embed_pos_rank, c.embed_dir_rank = self.embed_pos_rank, self.embed_dir_rank
        c.sdf_layer_count, c.sdf_layer_width = self.sdf_layer_count, self.sdf_layer_width
        c.col_layer_count, c.col_layer_width = self.col_layer_count, self.col_layer_width
        c.activation_type = L.ACT_IDS[self.activation_type]
        return self._fill_skips(c)

    def _param_tensors(self) -> List[Tensor]:
        """The layers' weights and biases, then the variance (packed too: the extra argument of the set_weights calls)."""
        return super()._param_tensors() + [self.variance]

    def _launch_forward(self, a: Tensor, b: Tensor, c, sampling_type, ray_radius: float, with_normal: bool) -> Dict[str, Tensor]:
        """The inference kernel on rays (sampling_type given) or explicit samples; called under no_grad."""
        if sampling_type is not None:
            return self.forward_rays(a, b, c, sampling_type, ray_radius, with_normal=with_normal)
        return self.forward(Sampling(a, b, a), with_normal=with_normal)

    def _forward_autograd(self, a: Tensor, b: Tensor, c, sampling_type, ray_radius: float, with_normal: bool) -> Dict[str, Tensor]:
        res = _NeusTrainFn.apply(self, a, b, c, sampling_type, float(ray_radius), with_normal, *self._param_tensors())
        out = {"sdf": res[0], "density": res[1], "color": res[2]}
        if with_normal:
            out["normal"] = res[3]
        return out

    def _shade_hits(self, hits: Tensor, pos: Tensor, dirs: Tensor, normal: Tensor, color: Tensor) -> None:
        """The exact normal of ``forward(with_normal=True)``, normalised (``unit_normals``), and the colour of the same
        call, stored by ray id."""
        p = pos[None]
        out = self.forward(Sampling(p, dirs[None], p), with_normal=True)
        idx = hits.long()
        normal.index_copy_(0, idx, unit_normals(out["normal"].reshape(-1, 3)))
        color.index_copy_(0, idx, out["color"].reshape(-1, 3))

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
        wants_grad = self._wants_grad()
        pos = L.require_cuda_f32(sampling.sample_pos, "sample_pos")
        sdir = L.require_cuda_f32(sampling.sample_dir, "sample_dir")
        B, S = pos.shape[0], pos.shape[1]
        if wants_grad:
            return self._forward_autograd(pos.reshape(B, S, 3), sdir.reshape(B, S, 3), None, None, 0.0, with_normal)
        device = pos.device
        out = self._outputs(B, S, device, with_normal)
        h = self._field(device)
        with torch.cuda.device(device):
            L.check(L.lib().neddf_neus_forward(h, L.ptr(pos), L.ptr(sdir), B * S, L.ptr(out["sdf"]), L.ptr(out["density"]),
                                               L.ptr(out["color"]), L.ptr(out.get("normal")), L.stream_ptr(device)),
                    "neus_forward")
        return out

    def forward_rays(self, ray_dir: Tensor, ray_orig: Tensor, dists: Tensor, sampling_type: str, ray_radius: float,
                     need_penalty: bool = True, need_aux: bool = True, need_color: bool = True, with_normal: bool = False) -> Dict[str, Tensor]:
        """Same network with the sample geometry fused into the kernel (what NeRFRender calls; this variant has
        neither penalties nor auxiliary fields, the flags are accepted for interface parity)."""
        wants_grad = self._wants_grad()
        ray_dir = L.require_cuda_f32(ray_dir, "ray_dir")
        ray_orig = L.require_cuda_f32(ray_orig, "ray_orig")
        dists = L.require_cuda_f32(dists, "dists")
        if wants_grad:
            return self._forward_autograd(ray_dir, ray_orig, dists, sampling_type, ray_radius, with_normal)
        B, S = dists.shape
        device = dists.device
        out = self._outputs(B, S, device, with_normal)
        h = self._field(device)
        with self._profiled(device, B * S), torch.cuda.device(device):
            L.check(L.lib().neddf_neus_forward_rays(h, L.ptr(ray_dir), L.ptr(ray_orig), L.ptr(dists), B, S,
                                                    L.SAMPLING_IDS[sampling_type], float(ray_radius), L.ptr(out["sdf"]),
                                                    L.ptr(out["density"]), L.ptr(out["color"]), L.ptr(out.get("normal")),
                                                    L.stream_ptr(device)), "neus_forward_rays")
        return out

    def forward_rays_segment(self, ray_dir: Tensor, ray_orig: Tensor, dists: Tensor, sampling_type: str, ray_radius: float,
                             edge0: int, seg_len: int, ray_index: Optional[Tensor], n_active: Optional[Tensor],
                             density: Tensor, color: Tensor) -> None:
        """One depth segment of the fine pass for early ray termination (neddf_neus_forward_rays_segment): samples
        [edge0, edge0 + seg_len) of the rays listed in ``ray_index[:n_active]`` (device tensors, None = all rays);
        density [B,E] and color [B,E,3] are scattered in place, equal bit for bit to what ``forward_rays`` gives there
        (the sdf and the normal are evaluated but not returned).  No-grad only."""
        self._refuse_autograd("forward_rays_segment")
        B, E = dists.shape
        device = dists.device
        h = self._field(device)
        # the executed count lives on the device (NeRFRender.termination_stats): no n_evaluations
        with self._profiled(device, None), torch.cuda.device(device):
            L.check(L.lib().neddf_neus_forward_rays_segment(
                h, L.ptr(ray_dir), L.ptr(ray_orig), L.ptr(dists), B, E, L.SAMPLING_IDS[sampling_type], float(ray_radius),
                int(edge0), int(seg_len), L.ptr(ray_index), L.ptr(n_active), L.ptr(density), L.ptr(color),
                L.stream_ptr(device)), "neus_forward_rays_segment")
