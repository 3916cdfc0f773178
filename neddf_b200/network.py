"""NeDDF field network: the reference's module surface over the CUDA megakernel.

Reference: neddf/network/neddf.py (NeDDF), neddf/network/base_neuralfield.py
(BaseNeuralField), neddf/nn_module/with_grad/linear.py:87-133 (LinearGradLayer parameters).

The module owns the same parameters under the same names/shapes as the reference
(``layers_ddf.{i}.weight`` [in,out] ...), so ``state_dict`` files are interchangeable.  All
arithmetic of ``forward`` happens in libneddf_b200.so (neddf_field_forward*); the parameters
are re-packed into kernel layout whenever their version counters change (optimiser steps
update them in place).
"""
import contextlib
import ctypes as C
import math
import warnings
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
from torch import Tensor, nn

from . import _lib as L
from ._host import KernelHandle, WeightGrad
from .ray import Sampling


class LinearGradLayer(nn.Module):
    """Parameter holder with the reference's layout: weight [in,out] xavier-normal, zero bias
    (nn_module/with_grad/linear.py:111-116).  The product computes y = xW + b, G = JW inside
    the fused field kernel, never layer by layer."""

    def __init__(self, input_ch: int = 128, output_ch: int = 128) -> None:
        super().__init__()
        self.input_ch, self.output_ch = input_ch, output_ch
        self.weight = nn.Parameter(torch.randn(input_ch, output_ch))
        self.bias = nn.Parameter(torch.randn(output_ch))
        nn.init.xavier_normal_(self.weight)
        nn.init.constant_(self.bias, 0.0)

    def forward(self, *a, **k):  # pragma: no cover
        raise NotImplementedError("neddf_b200 fuses all linear layers into the field megakernel; "
                                  "call NeDDF.forward instead")


class _FieldTrainFn(torch.autograd.Function):
    """Differentiable NeDDF.forward on rays + edge distances (training path).

    forward : neddf_field_forward_train - the fused megakernel of the module's engine (``net.engine``:
              tensor-core by default, "fp32" on request), keeping every layer's pre-activations.
    backward: neddf_field_backward does all sample-local work (activation second derivatives, heads,
              density, penalties, data-gradient GEMMs) and writes per-layer inputs X_l and
              pre-activation gradients G_l; the weight gradients gW_l = X_l^T G_l are tensor-core split-K
              GEMMs of this library (neddf_wgrad, csrc/wgrad.cu), bias gradients column sums
              (neddf_colsum_value_rows).
    Gradients flow to the module's parameters only (sample positions come from torch.rand / a
    no_grad resampling in the reference, nerf_render.py:131-166).
    """

    @staticmethod
    def forward(ctx, net, a, b, c, sampling_type, ray_radius, *params):
        """(a, b, c) = (ray_dir[B,3], ray_orig[B,3], dists[B,S]) with a sampling type, or the Sampling
        tensors (pos, dir, var)[B,S,3] when sampling_type is None."""
        from_rays = sampling_type is not None
        B, S = (c.shape if from_rays else a.shape[:2])
        n = B * S
        device = a.device
        n_hidden = (net.ddf_layer_count - 1) + (net.col_layer_count - 1)
        h = net._field(device)
        st = net._state_struct()
        save = torch.empty(n_hidden, n, 4, 256, device=device, dtype=torch.float32)
        density = torch.empty(B, S, device=device, dtype=torch.float32)
        color = torch.empty(B, S, 3, device=device, dtype=torch.float32)
        penalty = torch.empty(B, S, device=device, dtype=torch.float32)
        distance = torch.empty(B, S, device=device, dtype=torch.float32) if not from_rays else None
        aux = torch.empty(B, S, device=device, dtype=torch.float32) if not from_rays else None
        with torch.cuda.device(device):
            if from_rays:
                L.check(L.lib().neddf_field_forward_train(
                    h, C.byref(st), L.ptr(a), L.ptr(b), L.ptr(c), B, S, L.SAMPLING_IDS[sampling_type],
                    float(ray_radius), L.ptr(density), L.ptr(color), L.ptr(penalty), L.ptr(save),
                    net._engine_id(), L.stream_ptr(device)), "field_forward_train")
            else:
                L.check(L.lib().neddf_field_forward_train_samples(
                    h, C.byref(st), L.ptr(a), L.ptr(b), L.ptr(c), n, L.ptr(distance), L.ptr(density), L.ptr(color),
                    L.ptr(penalty), L.ptr(aux), L.ptr(save), net._engine_id(), L.stream_ptr(device)),
                    "field_forward_train_samples")
        ctx.net = net
        ctx.meta = (sampling_type, float(ray_radius),
                    (st.aux_grad_scale, st.distance_range_max, st.lowpass_alpha, tuple(st.penalty_weight)), (B, S))
        ctx.save_for_backward(a, b, c, save)
        if from_rays:
            return density, color, penalty
        ctx.mark_non_differentiable(distance, aux)
        return density, color, penalty, distance, aux

    @staticmethod
    def backward(ctx, g_density, g_color, g_penalty, *unused):
        net = ctx.net
        ga, gb_, gc_, save = ctx.saved_tensors
        sampling_type, ray_radius, stv, (B, S) = ctx.meta
        from_rays = sampling_type is not None
        n = B * S
        device = ga.device
        n_ddf, n_col = net.ddf_layer_count - 1, net.col_layer_count - 1
        n_hidden = n_ddf + n_col
        n_e0 = 6 * net.embed_pos_rank
        off_h = 6 * (net.embed_pos_rank + net.embed_dir_rank) + 3

        def prep(g, shape):
            if g is None:
                return torch.zeros(shape, device=device, dtype=torch.float32)
            return g.contiguous().to(torch.float32)

        g_density = prep(g_density, (B, S))
        g_color = prep(g_color, (B, S, 3))
        g_penalty = prep(g_penalty, (B, S))
        post = torch.empty(n_hidden, n, 4, 256, device=device, dtype=torch.float32)
        gpre = torch.empty(n_hidden, n, 4, 256, device=device, dtype=torch.float32)
        ghead_da = torch.empty(n, 4, 2, device=device, dtype=torch.float32)
        ghead_col = torch.empty(n, 4, 4, device=device, dtype=torch.float32)
        xes = torch.empty(n, 4, n_e0, device=device, dtype=torch.float32)
        xcol = torch.empty(n, 4, off_h, device=device, dtype=torch.float32)
        h = net._field(device)
        st = L.FieldState(stv[0], stv[1], stv[2], (C.c_float * L.N_PENALTY)(*stv[3]))
        with torch.cuda.device(device):
            if from_rays:
                L.check(L.lib().neddf_field_backward(
                    h, C.byref(st), L.ptr(ga), L.ptr(gb_), L.ptr(gc_), B, S, L.SAMPLING_IDS[sampling_type],
                    ray_radius, L.ptr(save), L.ptr(g_density), L.ptr(g_color), L.ptr(g_penalty), L.ptr(post),
                    L.ptr(gpre), L.ptr(ghead_da), L.ptr(ghead_col), L.ptr(xes), L.ptr(xcol), L.stream_ptr(device)),
                    "field_backward")
            else:
                L.check(L.lib().neddf_field_backward_samples(
                    h, C.byref(st), L.ptr(ga), L.ptr(gb_), L.ptr(gc_), n, L.ptr(save), L.ptr(g_density),
                    L.ptr(g_color), L.ptr(g_penalty), L.ptr(post), L.ptr(gpre), L.ptr(ghead_da), L.ptr(ghead_col),
                    L.ptr(xes), L.ptr(xcol), L.stream_ptr(device)), "field_backward_samples")

        # weight gradients gW = X^T G over the 4N rows (linear.py:76-79) and bias gradients (sum over the value
        # rows): tensor-core split-K GEMMs of this library (WeightGrad), written straight into the gradient tensors - no
        # vendor GEMM on the training path
        wg = WeightGrad(net, device, n)
        R = 4 * n
        grads = []
        with torch.cuda.device(device):
            for l in range(n_hidden):  # the weights are [in, out]: X^T G is the gradient as it stands
                if l == 0:
                    parts = [(xes, n_e0)]
                elif l < n_ddf:
                    parts = ([(xes, n_e0)] if (l - 1) in net.skips else []) + [(post[l - 1], 256)]
                elif l == n_ddf:
                    parts = [(xcol, off_h), (post[n_ddf - 1], 256)]
                else:
                    parts = [(post[l - 1], 256)]
                grads += wg.layer(parts, gpre[l], R, 4 * 256)
            # heads: gW^T [outs, 256] = ghead^T post (the 2- / 3-column head gradients are the A operand)
            gda_t = wg.empty(2, 256)
            wg.into(gda_t, 0, ghead_da, 2, 2, post[n_ddf - 1], R)
            gc_t = wg.empty(3, 256)
            wg.into(gc_t, 0, ghead_col, 4, 3, post[n_hidden - 1], R)
        b_da = ghead_da[:, 0, :].sum(0)
        grads += [gda_t[0].reshape(256, 1).contiguous(), b_da[0:1].contiguous(), gda_t[1].reshape(256, 1).contiguous(),
                  b_da[1:2].contiguous()]
        grads += [gc_t.t().contiguous(), ghead_col[:, 0, :3].sum(0)]
        return (None, None, None, None, None, None) + tuple(grads)


# network class name -> (field, level) of its surface: the level set ``extract_mesh`` meshes by default (``python -m
# neddf_b200.mesh``) and ``trace_surface`` traces (``NeRFRender.render_surface``).  NeDDF: the reference visualiser's
# iso-level of the distance field; NeuS: the SDF's zero set; NeRF has no canonical level.
LEVEL_DEFAULTS = {"NeDDF": ("distance", 0.0275), "NeuS": ("sdf", 0.0), "NeRF": ("density", None)}


class EngineRangeError(FloatingPointError):
    """The tensor-core engine left fp16 range under engine "auto"; the network has switched itself to the fp32 engine
    and the caller (NeRFRender) re-runs the call.  Explicit engines ("tc", "tc2") raise plain FloatingPointError."""


class BaseNeuralField(nn.Module):
    """neddf/network/base_neuralfield.py:11-79, plus the kernel plumbing the CUDA networks share: their C handles (one
    ``KernelHandle`` per kind in ``_HANDLES``: the forward handle, then the training one if any), the opt-in refusal of
    autograd and the CUDA-event bracket bench.py reads."""

    _HANDLES: Tuple[KernelHandle, ...] = ()
    _GRAD_REFUSAL: Optional[str] = None  # set for a network whose training backward is opt-in (``training_kernels``)

    def __init__(self) -> None:
        super().__init__()
        for h in self._HANDLES:
            h.reset(self)
        self._profile_events = None  # bench.py: list receiving (start, end, n_evaluations or None) CUDA events

    def _field(self, device: torch.device):
        """Forward handle with weights packed for the parameters' current values."""
        if device.type != "cuda":
            raise RuntimeError(f"neddf_b200.{type(self).__name__} runs on CUDA devices only: move the module with "
                               ".to('cuda') (the hot path has no CPU implementation)")
        return self._HANDLES[0].get(self, device)

    def _train_field(self, device: torch.device):
        """Handle of the training-backward kernel (NeRF, NeuS), re-packed like ``_field``'s."""
        return self._HANDLES[1].get(self, device)

    def _param_tensors(self) -> List[Tensor]:
        """The tensors the kernel packs are keyed on: weight and bias of every layer of ``_ordered_layers``."""
        return [t for l in self._ordered_layers() for t in (l.weight, l.bias)]

    def _fill_skips(self, cfg):
        if len(self.skips) > L.MAX_SKIPS:
            raise NotImplementedError("neddf_b200: more than 8 skip connections")
        cfg.n_skips = len(self.skips)
        for i, s in enumerate(self.skips):
            cfg.skips[i] = s
        return cfg

    def _release(self) -> None:
        for h in self._HANDLES:
            h.release(self)

    def __del__(self):
        try:
            self._release()
        except Exception:  # interpreter shutdown: torch internals may already be gone
            pass

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self.invalidate()  # .to()/.cuda() replaced the parameter storage
        return r

    def invalidate(self) -> None:
        """Force a re-pack of the kernel-layout weights on the next call.  Needed only after edits that
        bypass the parameters' version counters (``p.data.copy_(...)``, EMA swaps through ``.data``);
        optimiser steps, ``load_state_dict`` and ``.to()`` are detected automatically."""
        for h in self._HANDLES:
            setattr(self, h.names[2], None)

    # the kernel handles are process-local pointers: copies and pickles get fresh ones lazily
    def __getstate__(self):
        d = self.__dict__.copy()
        d.update({name: None for h in self._HANDLES for name in h.names})
        d["_profile_events"] = None
        d.pop("_wgrad_ws", None)
        return d

    def check_engine_status(self) -> None:
        """(fp32 kernel: no range checks to report)"""

    def _wants_grad(self) -> bool:
        """Autograd is recording and some parameter is trainable.  Without the opt-in that is refused."""
        if not (torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())):
            return False
        if self._GRAD_REFUSAL is not None and not self.training_kernels:
            raise NotImplementedError(self._GRAD_REFUSAL)
        return True

    def _refuse_autograd(self, what: str) -> None:
        """Raise when autograd is recording for a trainable parameter: ``what`` skips samples and has no gradient."""
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise RuntimeError(f"neddf_b200.{type(self).__name__}.{what} evaluates the samples of early ray termination "
                               "and has no gradient: call it under torch.no_grad() (render_image does)")

    @contextlib.contextmanager
    def _profiled(self, device: torch.device, n_evaluations: Optional[int]):
        """Brackets a launch with CUDA events appended to ``_profile_events`` when it is a list."""
        prof = self._profile_events
        if prof is None:
            yield
            return
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(torch.cuda.current_stream(device))
        yield
        e1.record(torch.cuda.current_stream(device))
        prof.append((e0, e1, n_evaluations))

    @property
    def device(self) -> torch.device:
        return next(self.parameters()).device

    def set_iter(self, iter: int) -> None:
        pass

    def voxelize(self, field_name: str = "density", cube_range: float = 1.1, cube_resolution: int = 64,
                 chunk: int = 65536) -> np.ndarray:
        """Dense-grid evaluation (base_neuralfield.py:49-79); same points in the same order as the reference, one
        device-to-host copy at the end."""
        return self._grid_volume(field_name, cube_range, cube_resolution, chunk).cpu().numpy()

    def _grid_volume(self, field_name: str, cube_range: float, cube_resolution: int, chunk: int = 65536) -> Tensor:
        """``voxelize``'s grid evaluated on the device: fp32 [n, n, n] on the module's device.

        The reference builds ``np.meshgrid(ids, ids, ids)`` ('xy' indexing) of ``ids = linspace(-r, r, n)`` and
        evaluates it in row-major order, so grid point (i, j, k) is at (x, y, z) = (ids[k], ids[i], ids[j]).  Here the
        positions of each chunk are gathered from the fp32 ``ids`` on the device, with direction (1, 0, 0) and zero
        variance, through ``self.forward`` in the module's current ``set_iter`` state; no host synchronisation."""
        n = int(cube_resolution)
        device = self.device
        with torch.set_grad_enabled(False):
            ids = self._grid_ids(cube_range, n)
            total = n ** 3
            out = torch.empty(total, dtype=torch.float32, device=device)
            for i in range(0, total, chunk):
                j = min(total, i + chunk)
                lin = torch.arange(i, j, device=device)
                out[i:j] = self._grid_values(field_name, ids, torch.stack([lin // (n * n), (lin // n) % n, lin % n], 1))
            return out.view(n, n, n)

    def _grid_ids(self, cube_range: float, n: int) -> Tensor:
        """``voxelize``'s axis coordinates ``linspace(-r, r, n)`` in fp32, on the module's device."""
        return torch.from_numpy(np.linspace(-cube_range, cube_range, n).astype(np.float32)).to(self.device)

    def _grid_values(self, field_name: str, ids: Tensor, idx: Tensor) -> Tensor:
        """The field at grid points ``idx`` [m, 3] (i, j, k) of ``voxelize``'s grid, [m] fp32: the point (x, y, z) =
        (ids[k], ids[i], ids[j]) gathered on the device, direction (1, 0, 0), zero variance, one ``forward``."""
        p = torch.stack([ids[idx[:, 2]], ids[idx[:, 0]], ids[idx[:, 1]]], 1)[None]
        dirs = torch.zeros_like(p)
        dirs[..., 0] = 1.0
        return self.forward(Sampling(p, dirs, torch.zeros_like(p)))[field_name].reshape(-1)

    def _band_mesh(self, field_name: str, threshold: float, cube_range: float, n: int, lipschitz: float,
                   normals: bool, chunk: int = 65536):
        """``narrow_band_marching_cubes`` over ``voxelize``'s grid, the points evaluated by ``_grid_values`` in chunks
        of ``chunk`` as ``_grid_volume`` evaluates them; band = L sqrt(3) 8 h in float64, rounded to fp32."""
        from .mesh import BRICK, narrow_band_marching_cubes
        h = 2.0 * float(cube_range) / (n - 1)
        band = float(np.float32(lipschitz * math.sqrt(3.0) * BRICK * h))
        with torch.set_grad_enabled(False), torch.cuda.device(self.device):
            ids = self._grid_ids(cube_range, n)

            def evaluate(idx: Tensor) -> Tensor:
                return torch.cat([self._grid_values(field_name, ids, idx[i:i + chunk])
                                  for i in range(0, idx.shape[0], chunk)])

            return narrow_band_marching_cubes(evaluate, n, threshold, band, normals=normals)

    # field -> sign of the colour pass's view direction relative to the vertex normal (which points toward increasing
    # value): -1 for a field that grows outward, +1 for one that grows inward, so the surface is seen from outside.
    # Only these fields can be meshed with_color.
    _MESH_VIEW_SIGN: Dict[str, float] = {}

    def extract_mesh(self, field_name: str, threshold: float, cube_range: float = 1.1, cube_resolution: int = 64,
                     with_color: bool = False, lipschitz: Optional[float] = None):
        """Triangle mesh of the level set ``field == threshold`` over ``voxelize``'s grid, on the module's device:
        (vertices [V,3] fp32, faces [F,3] int64).

        The grid is evaluated on the device (``_grid_volume``) and meshed by the marching-cubes kernels
        (``neddf_b200.mesh.marching_cubes``).  Vertices are returned in the camera frame: grid index (i, j, k) maps to
        (x, y, z) = (-r + k h, -r + i h, -r + j h) with h = 2r / (n - 1), computed in float64 and rounded to fp32.
        That map is a cyclic permutation of the axes, so the winding is kept: triangle normals point toward
        increasing field value, i.e. outward for ``distance`` / ``sdf`` and inward for ``density``.

        ``with_color=True`` returns (vertices, faces, normals [V,3] fp32, colors [V,3] fp32): the kernels' unit
        area-weighted vertex normals under the same axis permutation (exact: h is isotropic), and the field's
        ``color`` at every vertex, evaluated through ``forward`` in the module's current ``set_iter`` state with zero
        variance and a view direction looking at the surface from outside: ``-normal`` for ``distance`` / ``sdf``,
        ``+normal`` for ``density`` (NeDDF, NeRF).  Any other field raises ValueError.  Vertices and faces are the
        ``with_color=False`` ones bit for bit.

        ``lipschitz=L`` (finite, > 0; only the network's distance field, ``distance`` for NeDDF and ``sdf`` for NeuS)
        evaluates the grid only in a narrow band around the level set (``neddf_b200.mesh.narrow_band_marching_cubes``
        with band ``L sqrt(3) 8 h``), and ``cube_resolution`` may then be up to 2048.  If the field is L-Lipschitz on
        the grid, the result is the dense call's (``lipschitz=None``) bit for bit, in the same order; the bound is the
        caller's claim about its field and is not checked.

        The reference's visualiser writes its mesh in a scaled, half-voxel-shifted index space instead
        (fields_visualizer.py:546-547); that frame is not reproduced here."""
        from .mesh import BAND_MAX_DIM, MAX_DIM, marching_cubes
        n = int(cube_resolution)
        if n < 2:
            raise ValueError("extract_mesh: cube_resolution must be >= 2")
        if with_color and field_name not in self._MESH_VIEW_SIGN:
            raise ValueError(f"extract_mesh: with_color needs a field that is monotone across the surface; "
                             f"{type(self).__name__} supports {sorted(self._MESH_VIEW_SIGN)}, got {field_name!r}")
        if lipschitz is not None:
            lipschitz = float(lipschitz)
            if not (math.isfinite(lipschitz) and lipschitz > 0):
                raise ValueError(f"extract_mesh: lipschitz must be finite and > 0, got {lipschitz!r}")
            if self._TRACE_FIELD is None or field_name != self._TRACE_FIELD:
                raise ValueError(f"extract_mesh: the narrow band needs a distance field; {type(self).__name__} "
                                 f"{'has none' if self._TRACE_FIELD is None else 'has ' + repr(self._TRACE_FIELD)}, "
                                 f"got {field_name!r}")
            if n > BAND_MAX_DIM:
                raise ValueError(f"extract_mesh: cube_resolution must be in [2, {BAND_MAX_DIM}] with lipschitz, "
                                 f"got {n}")
            mesh = self._band_mesh(field_name, threshold, cube_range, n, lipschitz, with_color)
        else:
            if n > MAX_DIM:
                raise ValueError(f"extract_mesh: cube_resolution above {MAX_DIM} needs the narrow band: pass "
                                 f"lipschitz (a bound on the field's gradient norm), got {n}")
            volume = self._grid_volume(field_name, cube_range, n)
            mesh = marching_cubes(volume, threshold, normals=with_color)
        if with_color:
            vertices, faces, index_normals = mesh
        else:
            vertices, faces = mesh
        h = 2.0 * float(cube_range) / (n - 1)
        v = vertices.double()
        r = float(cube_range)
        world = torch.stack([-r + v[:, 2] * h, -r + v[:, 0] * h, -r + v[:, 1] * h], 1).float()
        if not with_color:
            return world, faces
        normals = index_normals[:, [2, 0, 1]]
        view_dir = -normals if self._MESH_VIEW_SIGN[field_name] < 0 else normals
        colors = self._vertex_colors(world, view_dir)
        if getattr(self, "engine", None) == "auto":
            try:
                self.check_engine_status()
            except EngineRangeError as e:  # engine "auto" left fp16 range: the colours again on the fp32 engine
                warnings.warn(str(e), RuntimeWarning)
                colors = self._vertex_colors(world, view_dir)
        return world, faces, normals, colors

    # the field whose values sphere tracing may step by (a distance or an SDF); None: the network cannot be traced
    _TRACE_FIELD: Optional[str] = None

    def surface_level(self, level: Optional[float] = None) -> float:
        """``level``, or the network's default surface level (``LEVEL_DEFAULTS``).  ValueError for a network without a
        distance field to trace (NeRF)."""
        if self._TRACE_FIELD is None:
            raise ValueError(f"{type(self).__name__} has no distance field: its surface cannot be sphere-traced")
        if level is None:
            level = LEVEL_DEFAULTS[type(self).__name__][1]
        level = float(level)
        if not np.isfinite(level) or abs(level) > float(np.finfo(np.float32).max):
            raise ValueError(f"trace_surface: level must be a finite fp32 value, got {level!r}")
        return level

    @staticmethod
    def _check_trace_args(near: float, far: float, max_steps: int) -> None:
        if not isinstance(max_steps, (int, np.integer)) or isinstance(max_steps, bool) or not 1 <= max_steps < 2 ** 31:
            raise ValueError(f"trace_surface: max_steps must be an integer >= 1, got {max_steps!r}")
        if not (np.isfinite(near) and np.isfinite(far) and 0.0 <= near < far):
            raise ValueError(f"trace_surface: need finite 0 <= near < far, got near={near!r}, far={far!r}")

    def trace_surface(self, ray_dir: Tensor, ray_orig: Tensor, near: float, far: float, level: float,
                      max_steps: int = 128) -> Dict[str, Tensor]:
        """First hit of the level set ``field == level`` along each ray by sphere tracing (csrc/surface.cu), under
        no_grad.  ``ray_dir`` (unit) / ``ray_orig`` [n,3] on the module's device.  Returns flat per-ray tensors:
        ``depth`` [n] (t of the hit; ``far`` on a miss), ``hit`` [n] bool, ``normal`` [n,3] (unit, toward increasing
        value; 0 on a miss), ``color`` [n,3] (the field's colour at the hit seen along the ray; 0 on a miss) and
        ``steps`` [n] int32 (field evaluations spent on the ray, normals and colour not counted).

        g(t) = field(o + t d) - level is evaluated through ``forward`` with point samples, zero variance and view
        direction d in the module's current ``set_iter`` state, as ``extract_mesh`` evaluates its grid.  From t = near:
        g >= EPS (1e-4) steps t += g (beyond far: miss), 0 <= g < EPS is a hit, g < 0 bisects the last step 8 times
        and hits at the near end of the bracket, so every hit has g >= 0.  g < 0 at t = near (the ray starts inside)
        and max_steps evaluations without a hit are misses.  One host read of the live count (4 bytes) per iteration:
        the point-query forwards take their sample count from the host.  Under engine "auto" the engine status is
        read once at the end; if the tensor-core engine left fp16 range the trace is run again on the fp32 engine."""
        level = self.surface_level(level)
        near, far = float(near), float(far)
        self._check_trace_args(near, far, max_steps)
        ray_dir = L.require_cuda_f32(ray_dir, "ray_dir")
        ray_orig = L.require_cuda_f32(ray_orig, "ray_orig")
        if ray_dir.dim() != 2 or ray_dir.shape[1] != 3 or ray_orig.shape != ray_dir.shape:
            raise ValueError(f"trace_surface: rays must be [n,3], got {tuple(ray_dir.shape)} / {tuple(ray_orig.shape)}")
        out = self._trace(ray_dir, ray_orig, near, far, level, int(max_steps))
        if getattr(self, "engine", None) == "auto":
            try:
                self.check_engine_status()
            except EngineRangeError as e:  # engine "auto" left fp16 range: trace again on the fp32 engine
                warnings.warn(str(e), RuntimeWarning)
                out = self._trace(ray_dir, ray_orig, near, far, level, int(max_steps))
        return out

    def _trace_values(self, pos: Tensor, dirs: Tensor) -> Tensor:
        """``forward`` of packed samples [m,3] with zero variance -> the traced field [m]."""
        p = pos[None]
        return self.forward(Sampling(p, dirs[None], torch.zeros_like(p)))[self._TRACE_FIELD].reshape(-1)

    def _trace(self, ray_dir: Tensor, ray_orig: Tensor, near: float, far: float, level: float,
               max_steps: int) -> Dict[str, Tensor]:
        lib = L.lib()
        n = ray_dir.shape[0]
        device = ray_dir.device
        f32, i32 = dict(device=device, dtype=torch.float32), dict(device=device, dtype=torch.int32)
        t, lo, hi = (torch.empty(n, **f32) for _ in range(3))
        state, steps, count = torch.empty(n, **i32), torch.empty(n, **i32), torch.empty(1, **i32)
        live = [torch.empty(n, **i32), torch.empty(n, **i32)]
        pos, dirs = torch.empty(n, 3, **f32), torch.empty(n, 3, **f32)
        normal, color = torch.zeros(n, 3, **f32), torch.zeros(n, 3, **f32)
        with torch.no_grad(), torch.cuda.device(device):
            stream = L.stream_ptr(device)
            L.check(lib.neddf_trace_init(L.ptr(ray_dir), L.ptr(ray_orig), n, near, L.ptr(t), L.ptr(lo), L.ptr(hi),
                                         L.ptr(state), L.ptr(steps), L.ptr(live[0]), L.ptr(pos), L.ptr(dirs), stream),
                    "trace_init")
            n_live, k = n, 0
            while n_live:  # every live ray spends one evaluation per pass, so at most max_steps passes
                values = self._trace_values(pos[:n_live], dirs[:n_live])
                L.check(lib.neddf_trace_step(L.ptr(values), L.ptr(live[k]), n_live, L.ptr(ray_dir), L.ptr(ray_orig),
                                             far, level, max_steps, L.ptr(t), L.ptr(lo), L.ptr(hi), L.ptr(state),
                                             L.ptr(steps), L.ptr(live[1 - k]), L.ptr(count), L.ptr(pos), L.ptr(dirs),
                                             stream), "trace_step")
                k = 1 - k
                n_live = int(count.item())
            hits = live[k]
            L.check(lib.neddf_trace_hits(L.ptr(ray_dir), L.ptr(ray_orig), n, L.ptr(t), L.ptr(state), L.ptr(hits),
                                         L.ptr(count), L.ptr(pos), L.ptr(dirs), stream), "trace_hits")
            n_hit = int(count.item())
            if n_hit:
                self._shade_hits(hits[:n_hit], pos[:n_hit], dirs[:n_hit], normal, color)
        return {"depth": t, "hit": state == L.TRACE_HIT, "normal": normal, "color": color, "steps": steps}

    def _shade_hits(self, hits: Tensor, pos: Tensor, dirs: Tensor, normal: Tensor, color: Tensor) -> None:
        """Normals and colours of the hit rays ``hits`` (packed hit points ``pos``, ray directions ``dirs``), stored by
        ray id.  Normals by central differences of the traced field (6 points per hit, h = 1e-4): the distance
        Jacobian the NeDDF kernels carry is not one of their outputs."""
        lib = L.lib()
        m = hits.shape[0]
        device = pos.device
        pts, pdirs = torch.empty(6 * m, 3, device=device), torch.empty(6 * m, 3, device=device)
        stream = L.stream_ptr(device)
        L.check(lib.neddf_trace_fd_points(L.ptr(pos), L.ptr(dirs), m, L.ptr(pts), L.ptr(pdirs), stream), "trace_fd_points")
        values = self._trace_values(pts, pdirs)
        L.check(lib.neddf_trace_fd_normals(L.ptr(values), L.ptr(pos), L.ptr(hits), m, L.ptr(normal), stream),
                "trace_fd_normals")
        color.index_copy_(0, hits.long(), self._vertex_colors(pos, dirs))

    def _vertex_colors(self, points: Tensor, view_dir: Tensor, chunk: int = 65536) -> Tensor:
        """``forward(Sampling(points, view_dir, 0))["color"]`` [V,3] in chunks, with no host synchronisation."""
        with torch.set_grad_enabled(False):
            out = torch.empty(points.shape[0], 3, dtype=torch.float32, device=points.device)
            for i in range(0, points.shape[0], chunk):
                p = points[None, i:i + chunk]
                s = Sampling(p, view_dir[None, i:i + chunk], torch.zeros_like(p))
                out[i:i + chunk] = self.forward(s)["color"].reshape(-1, 3)
            return out


class NeDDF(BaseNeuralField):
    """Drop-in for neddf.network.NeDDF (neddf/network/neddf.py:21-326)."""

    _MESH_VIEW_SIGN = {"distance": -1.0, "density": 1.0}  # distance grows outward, density inward
    _HANDLES = (KernelHandle("neddf_field"),)
    _TRACE_FIELD = "distance"

    def __init__(
        self,
        embed_pos_rank: int = 10,
        embed_dir_rank: int = 4,
        ddf_layer_count: int = 8,
        ddf_layer_width: int = 256,
        col_layer_count: int = 8,
        col_layer_width: int = 256,
        activation_type: str = "tanhExp",
        density_activation_type: str = "ReLU",
        d_near: float = 0.01,
        lowpass_alpha_offset: float = 10.0,
        skips: Optional[List[int]] = None,
        penalty_weight: Optional[Dict[str, float]] = None,
    ) -> None:
        super().__init__()
        input_ddf_dim = embed_pos_rank * 6
        input_col_dim = (embed_pos_rank + embed_dir_rank) * 6 + 3 + ddf_layer_width
        if skips is None:
            skips = [4]
        self.skips = [int(s) for s in skips]
        if activation_type not in L.ACT_IDS or density_activation_type not in L.ACT_IDS:
            raise KeyError(f"unknown activation {activation_type!r}/{density_activation_type!r}")  # neddf.py:107-118
        self.activation_type = activation_type
        self.density_activation_type = density_activation_type
        self.embed_pos_rank, self.embed_dir_rank = int(embed_pos_rank), int(embed_dir_rank)
        self.ddf_layer_count, self.col_layer_count = int(ddf_layer_count), int(col_layer_count)
        self.ddf_layer_width, self.col_layer_width = int(ddf_layer_width), int(col_layer_width)

        # identical construction order and shapes to neddf.py:129-145
        layers_ddf = [LinearGradLayer(input_ddf_dim, ddf_layer_width)]
        for layer_id in range(ddf_layer_count - 2):
            extra = input_ddf_dim if layer_id in self.skips else 0
            layers_ddf.append(LinearGradLayer(ddf_layer_width + extra, ddf_layer_width))
        layers_col = [LinearGradLayer(input_col_dim, col_layer_width)]
        for _ in range(col_layer_count - 2):
            layers_col.append(LinearGradLayer(col_layer_width, col_layer_width))
        self.layers_ddf = nn.ModuleList(layers_ddf)
        self.layers_col = nn.ModuleList(layers_col)
        self.layer_ddf_out = LinearGradLayer(ddf_layer_width, 1)
        self.layer_aux_out = LinearGradLayer(ddf_layer_width, 1)
        self.layer_col_out = LinearGradLayer(ddf_layer_width, 3)

        self.d_near = float(d_near)
        self.aux_grad_scale = 1.1
        self.distance_range_max = 2.0
        self.lowpass_alpha_offset = float(lowpass_alpha_offset)
        self.lowpass_alpha = float(lowpass_alpha_offset)
        if penalty_weight is None:
            penalty_weight = {"constraints_aux_grad": 0.05, "constraints_dDdt": 0.05, "constraints_color": 0.01,
                              "range_distance": 1.0, "range_aux_grad": 1.0}
        self.penalty_weight = {k: float(v) for k, v in dict(penalty_weight).items()}

        # kernel-side state
        self.engine = "auto"          # "auto" | "fp32" | "tc" | "tc2"
        self._range_fallback = False  # "auto" met an activation outside fp16 range: it resolves to fp32 from then on

    def resolved_engine(self, device=None) -> str:
        """Engine that will actually run for ``self.engine`` ("fp32" or "tc")."""
        h = self._field(torch.device(device) if device is not None else self.device)
        rc = L.check(L.lib().neddf_field_resolve_engine(h, self._engine_id()), "resolve_engine")
        return {1: "fp32", 2: "tc", 3: "tc2"}[rc]

    def _engine_id(self) -> int:
        """ABI engine id of the next launch: ``self.engine``, except that "auto" stays on the fp32 engine once the
        tensor-core engine has reported an activation outside fp16 range for this network (check_engine_status)."""
        return L.ENGINE_IDS["fp32" if (self._range_fallback and self.engine == "auto") else self.engine]

    # ------------------------------------------------------------------ kernel plumbing --
    def _ordered_layers(self) -> List[LinearGradLayer]:
        return list(self.layers_ddf) + list(self.layers_col) + [self.layer_ddf_out, self.layer_aux_out, self.layer_col_out]

    def _config_struct(self) -> L.FieldConfig:
        c = L.FieldConfig()
        c.embed_pos_rank, c.embed_dir_rank = self.embed_pos_rank, self.embed_dir_rank
        c.ddf_layer_count, c.ddf_layer_width = self.ddf_layer_count, self.ddf_layer_width
        c.col_layer_count, c.col_layer_width = self.col_layer_count, self.col_layer_width
        c.activation_type = L.ACT_IDS[self.activation_type]
        c.density_activation_type = L.ACT_IDS[self.density_activation_type]
        c.d_near = self.d_near
        self._fill_skips(c)
        for i, k in enumerate(L.PENALTY_KEYS):  # absent key -> unweighted, neddf.py:296-299
            c.penalty_weight[i] = self.penalty_weight.get(k, 1.0)
        return c

    def _state_struct(self) -> L.FieldState:
        """Per-call scalars: the warm-up schedule and the penalty weights, both read from the module on
        every forward like the reference does (neddf.py:296-299: absent key -> unweighted)."""
        pw = (C.c_float * L.N_PENALTY)(*[float(self.penalty_weight.get(k, 1.0)) for k in L.PENALTY_KEYS])
        return L.FieldState(float(self.aux_grad_scale), float(self.distance_range_max), float(self.lowpass_alpha), pw)

    # ------------------------------------------------------------------------- forward --
    def forward(self, sampling: Sampling) -> Dict[str, Tensor]:
        """NeDDF.forward (neddf.py:162-309): Sampling[B,S,3] -> distance, density, color,
        fields_penalty, aux_grad.  Under autograd: the differentiable fp32 path (gradients to the
        parameters through density / color / fields_penalty; distance and aux_grad are returned
        without a graph - no loss of the reference consumes them)."""
        pos = sampling.sample_pos
        B, S = pos.shape[0], pos.shape[1]
        if self._wants_grad():
            p3 = L.require_cuda_f32(pos.reshape(B, S, 3), "sample_pos")
            d3 = L.require_cuda_f32(sampling.sample_dir.reshape(B, S, 3), "sample_dir")
            v3 = L.require_cuda_f32(sampling.diag_variance.reshape(B, S, 3), "diag_variance")
            d, c, pnl, dist, aux = _FieldTrainFn.apply(self, p3, d3, v3, None, 0.0, *self._param_tensors())
            return {"distance": dist, "density": d, "color": c, "fields_penalty": pnl, "aux_grad": aux}
        device = pos.device
        # reshape, not view: accept the expanded tensors the reference's point sampler returns
        p3 = L.require_cuda_f32(pos.reshape(-1, 3), "sample_pos")
        d3 = L.require_cuda_f32(sampling.sample_dir.reshape(-1, 3), "sample_dir")
        v3 = L.require_cuda_f32(sampling.diag_variance.reshape(-1, 3), "diag_variance")
        n = B * S
        out = {
            "distance": torch.empty(B, S, device=device, dtype=torch.float32),
            "density": torch.empty(B, S, device=device, dtype=torch.float32),
            "color": torch.empty(B, S, 3, device=device, dtype=torch.float32),
            "fields_penalty": torch.empty(B, S, device=device, dtype=torch.float32),
            "aux_grad": torch.empty(B, S, device=device, dtype=torch.float32),
        }
        h = self._field(device)
        st = self._state_struct()
        with torch.cuda.device(device):
            L.check(L.lib().neddf_field_forward(
                h, C.byref(st), L.ptr(p3), L.ptr(d3), L.ptr(v3), n, L.ptr(out["distance"]), L.ptr(out["density"]),
                L.ptr(out["color"]), L.ptr(out["fields_penalty"]), L.ptr(out["aux_grad"]), L.OUT_FULL,
                self._engine_id(), L.stream_ptr(device)), "field_forward")
        return out

    def forward_rays(self, ray_dir: Tensor, ray_orig: Tensor, dists: Tensor, sampling_type: str, ray_radius: float,
                     need_penalty: bool = True, need_aux: bool = True, need_color: bool = True) -> Dict[str, Tensor]:
        """Same network with the sample geometry fused into the kernel prologue (no [N,3]
        Sampling tensors in HBM).  Used by NeRFRender.  Under autograd (training) it runs the
        differentiable fp32 path (_FieldTrainFn) and returns density / color / fields_penalty.
        ``need_color=False`` (with ``need_penalty=False``) leaves "color" out: the tensor-core engines then skip
        the colour trunk, which is what an image's coarse pass wants (only its densities reach the image)."""
        ray_dir = L.require_cuda_f32(ray_dir, "ray_dir")
        ray_orig = L.require_cuda_f32(ray_orig, "ray_orig")
        dists = L.require_cuda_f32(dists, "dists")
        if self._wants_grad():
            d, c, pnl = _FieldTrainFn.apply(self, ray_dir, ray_orig, dists, sampling_type, ray_radius,
                                            *self._param_tensors())
            return {"density": d, "color": c, "fields_penalty": pnl}
        B, S = dists.shape
        device = dists.device
        out = {"density": torch.empty(B, S, device=device, dtype=torch.float32)}
        if need_color or need_penalty:
            out["color"] = torch.empty(B, S, 3, device=device, dtype=torch.float32)
        if need_penalty:
            out["fields_penalty"] = torch.empty(B, S, device=device, dtype=torch.float32)
        if need_aux:
            out["distance"] = torch.empty(B, S, device=device, dtype=torch.float32)
            out["aux_grad"] = torch.empty(B, S, device=device, dtype=torch.float32)
        h = self._field(device)
        st = self._state_struct()
        with self._profiled(device, B * S), torch.cuda.device(device):
            L.check(L.lib().neddf_field_forward_rays(
                h, C.byref(st), L.ptr(ray_dir), L.ptr(ray_orig), L.ptr(dists), B, S, L.SAMPLING_IDS[sampling_type],
                float(ray_radius), L.ptr(out.get("distance")), L.ptr(out["density"]), L.ptr(out.get("color")),
                L.ptr(out.get("fields_penalty")), L.ptr(out.get("aux_grad")),
                L.OUT_FULL if need_penalty else L.OUT_EVAL, self._engine_id(), L.stream_ptr(device)),
                "field_forward_rays")
        return out

    def forward_rays_segment(self, ray_dir: Tensor, ray_orig: Tensor, dists: Tensor, sampling_type: str, ray_radius: float,
                             edge0: int, seg_len: int, ray_index: Optional[Tensor], n_active: Optional[Tensor],
                             density: Tensor, color: Tensor) -> None:
        """One depth segment of the fine pass for early ray termination (neddf_field_forward_rays_segment):
        samples [edge0, edge0 + seg_len) of the rays listed in ``ray_index[:n_active]`` (device tensors, None =
        all rays); results are scattered into ``density`` [B,E] / ``color`` [B,E,3] in place.  No-grad only."""
        B, E = dists.shape
        device = dists.device
        h = self._field(device)
        st = self._state_struct()
        # the executed count lives on the device (NeRFRender.termination_stats): no n_evaluations
        with self._profiled(device, None), torch.cuda.device(device):
            L.check(L.lib().neddf_field_forward_rays_segment(
                h, C.byref(st), L.ptr(ray_dir), L.ptr(ray_orig), L.ptr(dists), B, E, L.SAMPLING_IDS[sampling_type],
                float(ray_radius), int(edge0), int(seg_len), L.ptr(ray_index), L.ptr(n_active), L.ptr(density),
                L.ptr(color), self._engine_id(), L.stream_ptr(device)), "field_forward_rays_segment")

    def check_engine_status(self) -> None:
        """Read-and-clear the engine's device status word (one sync).  Raises if the tensor-core
        engine met an activation outside fp16 range (its operands are fp16 hi+lo pairs)."""
        if self._handle is None:
            return
        v = C.c_int32(0)
        dev = self._handle_device
        with torch.cuda.device(dev):
            L.check(L.lib().neddf_field_status(self._handle, C.byref(v), L.stream_ptr(dev)), "field_status")
        if v.value & 4:
            if self.engine == "auto" and not self._range_fallback:
                self._range_fallback = True
                raise EngineRangeError(
                    "neddf_b200: tensor-core engine saw |activation| > 65504 (fp16 range of its split operands); "
                    "engine 'auto' now resolves to the fp32 engine for this network and the call is re-run")
            raise FloatingPointError(
                "neddf_b200: tensor-core engine saw |activation| > 65504 (fp16 range of its split operands); "
                "results of the last calls are invalid - use set_engine('fp32') or 'auto' for this network")

    def set_iter(self, iter: int) -> None:
        """Warm-up schedule (neddf.py:311-326); -1 = evaluation."""
        if iter == -1:
            self.aux_grad_scale = 1.1
            self.distance_range_max = 2.0
            self.lowpass_alpha = float(self.embed_pos_rank)
        else:
            self.aux_grad_scale = min(1.1, max(0.01, 0.0001 * iter))
            self.distance_range_max = min(2.0, 2.0 + 0.0001 * iter)
            self.lowpass_alpha = self.lowpass_alpha_offset + 0.001 * iter
