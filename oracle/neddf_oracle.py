"""CPU oracle for the NeDDF volumetric-rendering hot path.

TEST INFRASTRUCTURE ONLY.  This file is a functional torch-CPU restatement of the
reference algorithm (ueda0319/neddf @ f71838ea); it exists so that the CUDA path can
be checked on machines where /root/reference is absent (the GPU box).  Only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs may import it.  Nothing under ``neddf_b200/`` imports
it, and the product raises if its CUDA library is missing - there is no CPU
fallback.

Parity pin: this restatement is checked against the real reference, executed in
the build container by ``tests/golden/make_golden.py`` (which imports
``/root/reference`` and records inputs/outputs into ``tests/golden/*.npz``), by
``tests/test_oracle_golden.py``.

The NeRF and NeuS field variants (end of this file) are pinned the same way: ``make_nerf_golden.py`` /
``make_neus_golden.py`` run the reference's own networks inside its NeRFRender, ``tests/test_nerf_oracle.py`` /
``tests/test_neus_oracle.py`` hold ``nerf_forward`` / ``neus_forward`` to 2e-6 of them.

Every function cites the reference file:line it restates (paths relative to the
reference root).  All tensors are [rays, samples, ...] row-major; ``dtype`` may be
float32 (parity target) or float64 (arbiter for ill-conditioned samples).

A "sample row" convention used throughout: for every sample the network carries the
activation vector ``x[C]`` and the forward-mode Jacobian ``J[3, C]`` (d/dx, d/dy,
d/dz of every channel with respect to the sample position).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Tuple

import torch
from torch import Tensor

# --------------------------------------------------------------------------------------
# configuration containers (mirror the reference constructor arguments)
# --------------------------------------------------------------------------------------

DEFAULT_PENALTY_WEIGHT = {  # neddf/network/neddf.py:151-158
    "constraints_aux_grad": 0.05,
    "constraints_dDdt": 0.05,
    "constraints_color": 0.01,
    "range_distance": 1.0,
    "range_aux_grad": 1.0,
}


@dataclass
class FieldConfig:
    """Constructor arguments of NeDDF (neddf/network/neddf.py:52-66)."""

    embed_pos_rank: int = 10
    embed_dir_rank: int = 4
    ddf_layer_count: int = 8
    ddf_layer_width: int = 256
    col_layer_count: int = 8
    col_layer_width: int = 256
    activation_type: str = "tanhExp"
    density_activation_type: str = "ReLU"
    d_near: float = 0.01
    lowpass_alpha_offset: float = 10.0
    skips: Optional[List[int]] = None
    penalty_weight: Optional[Dict[str, float]] = None

    def __post_init__(self) -> None:
        if self.skips is None:
            self.skips = [4]
        if self.penalty_weight is None:
            self.penalty_weight = dict(DEFAULT_PENALTY_WEIGHT)

    @staticmethod
    def from_dict(d: Dict) -> "FieldConfig":
        d = {k: v for k, v in dict(d).items() if k != "_target_"}
        if d.get("skips") is not None:
            d["skips"] = [int(s) for s in d["skips"]]
        if d.get("penalty_weight") is not None:
            d["penalty_weight"] = {k: float(v) for k, v in dict(d["penalty_weight"]).items()}
        return FieldConfig(**d)


@dataclass
class FieldState:
    """Warm-up scalars set by NeDDF.set_iter (neddf/network/neddf.py:311-326)."""

    aux_grad_scale: float = 1.1
    distance_range_max: float = 2.0
    lowpass_alpha: float = 10.0

    @staticmethod
    def at_iter(cfg: FieldConfig, it: int) -> "FieldState":
        if it == -1:  # neddf.py:319-322
            return FieldState(1.1, 2.0, float(cfg.embed_pos_rank))
        return FieldState(  # neddf.py:323-326
            min(1.1, max(0.01, 0.0001 * it)),
            min(2.0, 2.0 + 0.0001 * it),
            cfg.lowpass_alpha_offset + 0.001 * it,
        )


@dataclass
class RenderConfig:
    """Constructor arguments of NeRFRender (neddf/render/nerf_render.py:40-50)."""

    sample_coarse: int = 128
    sample_fine: int = 128
    dist_near: float = 2.0
    dist_far: float = 6.0
    max_dist: float = 6.0
    use_coarse_network: bool = True
    sampling_type: str = "point"

    @staticmethod
    def from_dict(d: Dict) -> "RenderConfig":
        d = {k: v for k, v in dict(d).items() if k not in ("_target_", "network_config")}
        return RenderConfig(**d)


@dataclass
class CameraPose:
    """What create_rays reads from a Camera (neddf/camera/camera.py:155-171)."""

    R: Tensor  # [3,3]
    T: Tensor  # [3]
    fx: float
    fy: float
    cx: float
    cy: float


MatMul = Callable[[Tensor, Tensor], Tensor]

# --------------------------------------------------------------------------------------
# parameter initialisation (for seeded random networks)
# --------------------------------------------------------------------------------------


def layer_shapes(cfg: FieldConfig) -> List[Tuple[str, int, int]]:
    """Names and [in,out] shapes of the 13 linear layers (neddf/network/neddf.py:88-145)."""
    in_ddf = cfg.embed_pos_rank * 6
    in_col = (cfg.embed_pos_rank + cfg.embed_dir_rank) * 6 + 3 + cfg.ddf_layer_width
    shapes = [("layers_ddf.0", in_ddf, cfg.ddf_layer_width)]
    for lid in range(cfg.ddf_layer_count - 2):
        extra = in_ddf if lid in cfg.skips else 0
        shapes.append((f"layers_ddf.{lid + 1}", cfg.ddf_layer_width + extra, cfg.ddf_layer_width))
    shapes.append(("layers_col.0", in_col, cfg.col_layer_width))
    for lid in range(cfg.col_layer_count - 2):
        shapes.append((f"layers_col.{lid + 1}", cfg.col_layer_width, cfg.col_layer_width))
    shapes.append(("layer_ddf_out", cfg.ddf_layer_width, 1))
    shapes.append(("layer_aux_out", cfg.ddf_layer_width, 1))
    shapes.append(("layer_col_out", cfg.ddf_layer_width, 3))
    return shapes


def init_params(cfg: FieldConfig, seed: int, bias_std: float = 0.0) -> Dict[str, Tensor]:
    """Xavier-normal weights [in,out], zero bias (neddf/nn_module/with_grad/linear.py:113-116).

    ``bias_std`` > 0 perturbs the biases so that tests exercise the bias path.
    The random stream is this oracle's own (not the reference's), so goldens carry their
    weights explicitly.
    """
    g = torch.Generator().manual_seed(seed)
    out: Dict[str, Tensor] = {}
    for name, cin, cout in layer_shapes(cfg):
        std = math.sqrt(2.0 / (cin + cout))
        out[name + ".weight"] = torch.randn(cin, cout, generator=g) * std
        out[name + ".bias"] = torch.randn(cout, generator=g) * bias_std
    return out


# --------------------------------------------------------------------------------------
# NN primitives with forward-mode Jacobian
# --------------------------------------------------------------------------------------


def linear_jac(x: Tensor, J: Tensor, W: Tensor, b: Tensor, mm: Optional[MatMul] = None):
    """y = x W + b, G = J W with W stored [in,out] (nn_module/with_grad/linear.py:40-43)."""
    mm = mm or torch.matmul
    return mm(x, W) + b.unsqueeze(0), mm(J, W)


def act_tanhexp(x: Tensor, J: Tensor, threshold: float = 20.0):
    """x*tanh(exp x) with first derivative applied to J (nn_module/with_grad/tanh_exp.py:38-48)."""
    big = x > threshold
    ex = torch.exp(x)
    tx = torch.tanh(ex)
    y = torch.where(big, x, x * tx)
    d1 = torch.where(big, torch.ones_like(x), tx - x * ex * (tx * tx - 1))
    return y, d1.unsqueeze(1) * J


def act_relu(x: Tensor, J: Tensor):
    """nn_module/with_grad/relu.py:15-39 (slope 0 for x<0... mask is x<0, so f'(0)=1)."""
    s = torch.where(x < 0, torch.zeros_like(x), torch.ones_like(x))
    return x * s, J * s.unsqueeze(1)


def act_leaky_relu(x: Tensor, J: Tensor):
    """nn_module/with_grad/leaky_relu.py:36-39 (slope 0.01 for x<0)."""
    s = torch.where(x < 0, torch.full_like(x, 0.01), torch.ones_like(x))
    return x * s, J * s.unsqueeze(1)


def act_softplus(x: Tensor, J: Tensor, threshold: float = 20.0):
    """log(1+exp x), f' = 1/(1+exp(-x)) (nn_module/with_grad/softplus.py:38-48)."""
    big = x > threshold
    y = torch.where(big, x, torch.log(1.0 + torch.exp(x)))
    d1 = torch.where(big, torch.ones_like(x), 1.0 / (1.0 + torch.exp(-x)))
    return y, d1.unsqueeze(1) * J


def act_sigmoid(x: Tensor, J: Tensor):
    """(1+tanh(x/2))/2, f' = t(1-t) (nn_module/with_grad/sigmoid.py:38-43)."""
    t = (1.0 + torch.tanh(x * 0.5)) * 0.5
    d1 = t * (1 - t)
    return t, d1.unsqueeze(1) * J


HIDDEN_ACT = {"tanhExp": act_tanhexp, "ReLU": act_relu, "LeakyReLU": act_leaky_relu}


def density_act(name: str, x: Tensor) -> Tensor:
    """Plain activations selectable as density_activation (neddf/network/neddf.py:107-118)."""
    if name == "ReLU":
        return torch.relu(x)
    if name == "LeakyReLU":
        return torch.nn.functional.leaky_relu(x)  # slope 0.01
    if name == "tanhExp":  # nn_module/tanh_exp.py:26-31
        return torch.where(x > 20.0, x, x * torch.tanh(torch.exp(x)))
    raise ValueError(name)


def lowpass_scale(embed_dim: int, alpha: float, dtype=torch.float32) -> Tensor:
    """Per-frequency window [E] (nn_module/with_grad/positional_encoding.py:137-157)."""
    if alpha >= embed_dim:
        return torch.ones(embed_dim, dtype=dtype)
    s = torch.ones(embed_dim, dtype=dtype)
    k = int(alpha)
    s[k] = 0.5 * (1 - math.cos(math.pi * (alpha - k))) + 1e-7
    if k + 1 < embed_dim:
        s[k + 1:] = 1e-7
    return s


def pe_jacobian(pos: Tensor, scale: Tensor, embed_dim: int):
    """Positional encoding of positions with the analytic Jacobian for J_in = I.

    Channel order is [sin(e0:x,y,z), sin(e1:x,y,z) ... | cos(...)], i.e. channel
    e*3+d holds frequency 2^e of coordinate d
    (nn_module/with_grad/positional_encoding.py:65-87).
    """
    n = pos.shape[0]
    freq = (2.0 ** torch.arange(embed_dim, dtype=pos.dtype)).reshape(1, embed_dim, 1)
    p = (freq * pos.reshape(n, 1, 3)).reshape(n, embed_dim * 3)
    sp, cp = torch.sin(p), torch.cos(p)
    y = torch.cat([scale * sp, scale * cp], 1)
    # d p[e*3+d] / d pos_i = 2^e * (i == d)
    sel = torch.eye(3, dtype=pos.dtype).reshape(1, 3, 1, 3).expand(1, 3, embed_dim, 3)
    sel = sel.reshape(1, 3, embed_dim * 3)
    fs = (freq.expand(1, embed_dim, 3).reshape(1, 1, embed_dim * 3) * scale.unsqueeze(1)) * sel
    G = torch.cat([fs * cp.unsqueeze(1), -fs * sp.unsqueeze(1)], 2)
    return y, G


def pe_plain(v: Tensor, embed_dim: int) -> Tensor:
    """Positional encoding without Jacobian, unit scale (nn_module/positional_encoding.py:37-65)."""
    n = v.shape[0]
    freq = (2.0 ** torch.arange(embed_dim, dtype=v.dtype)).reshape(1, embed_dim, 1)
    p = (freq * v.reshape(n, 1, 3)).reshape(n, embed_dim * 3)
    return torch.cat([torch.sin(p), torch.cos(p)], 1)


def pe_weights(var: Tensor, embed_dim: int) -> Tensor:
    """exp(-0.5 * (2^e)^2 * var_d), channel e*3+d (neddf/ray/sampling.py:58-71)."""
    n = var.shape[0]
    fsq = ((2.0 ** torch.arange(embed_dim, dtype=var.dtype)) ** 2).reshape(1, embed_dim, 1)
    return torch.exp(-0.5 * (fsq * var.reshape(n, 1, 3)).reshape(n, embed_dim * 3))


# --------------------------------------------------------------------------------------
# the field network
# --------------------------------------------------------------------------------------


def field_forward(
    P: Dict[str, Tensor],
    cfg: FieldConfig,
    st: FieldState,
    pos: Tensor,
    dirs: Tensor,
    var: Tensor,
    mm: Optional[MatMul] = None,
    taps: Optional[Dict[str, Tensor]] = None,
) -> Dict[str, Tensor]:
    """NeDDF.forward (neddf/network/neddf.py:162-309) on a [B,S,3] block of samples.

    ``taps`` (optional dict) receives intermediates for per-stage parity tests.
    """
    B, S = pos.shape[0], pos.shape[1]
    n = B * S
    dt = pos.dtype
    x3, d3, v3 = pos.reshape(n, 3), dirs.reshape(n, 3), var.reshape(n, 3)
    E = cfg.embed_pos_rank
    act = HIDDEN_ACT[cfg.activation_type]

    # neddf.py:193-199 : scales for the two position encodings
    s_grad = (2.0 / (2.0 ** torch.arange(E, dtype=dt))).reshape(E, 1).expand(E, 3).reshape(1, 3 * E)
    s_low = lowpass_scale(E, st.lowpass_alpha, dt).reshape(E, 1).expand(E, 3).reshape(1, 3 * E)
    w_pe = pe_weights(v3, E)
    es, Jes = pe_jacobian(x3, s_grad * s_low * w_pe, E)  # neddf.py:200-204
    e0, Je0 = pe_jacobian(x3, s_low * w_pe, E)  # neddf.py:205-209
    ed = pe_plain(d3, cfg.embed_dir_rank)  # neddf.py:210
    if taps is not None:
        taps.update(embed_pos_scaled=es, embed_pos_scaled_J=Jes, embed_pos=e0, embed_pos_J=Je0, embed_dir=ed)

    # distance trunk, neddf.py:212-219
    h, hJ = es, Jes
    for lid in range(cfg.ddf_layer_count - 1):
        h, hJ = linear_jac(h, hJ, P[f"layers_ddf.{lid}.weight"], P[f"layers_ddf.{lid}.bias"], mm)
        if taps is not None:
            taps[f"ddf{lid}_pre"] = h
        h, hJ = act(h, hJ)
        if taps is not None:
            taps[f"ddf{lid}_x"], taps[f"ddf{lid}_J"] = h, hJ
        if lid in cfg.skips:
            h = torch.cat([es, h], 1)
            hJ = torch.cat([Jes, hJ], 2)

    # heads, neddf.py:220-230
    ddf_out, ddf_outJ = linear_jac(h, hJ, P["layer_ddf_out.weight"], P["layer_ddf_out.bias"], mm)
    sp, spJ = act_softplus(ddf_out, ddf_outJ)
    distance = sp + cfg.d_near
    grad_d = spJ[:, :, 0]
    aux_out, aux_outJ = linear_jac(h, hJ, P["layer_aux_out.weight"], P["layer_aux_out.bias"], mm)
    sg, sgJ = act_sigmoid(aux_out, aux_outJ)
    aux = st.aux_grad_scale * sg
    aux_gg = st.aux_grad_scale * sgJ[:, :, 0]

    # distance -> density, neddf.py:232-241
    grad_norm = torch.linalg.vector_norm(grad_d, dim=1, keepdim=True)
    dDdt = torch.linalg.vector_norm(torch.cat([grad_d, aux], 1), dim=1, keepdim=True)
    dist_inv = torch.reciprocal(distance)
    density = density_act(cfg.density_activation_type, dist_inv * (1 - dDdt))
    normal = torch.reciprocal(grad_norm + 1e-7) * grad_d

    # colour trunk, neddf.py:243-257
    c = torch.cat([e0, ed, normal.detach(), h], 1)
    cJ = torch.cat([Je0, torch.zeros(n, 3, ed.shape[1] + 3, dtype=dt), hJ], 2)
    for lid in range(cfg.col_layer_count - 1):
        c, cJ = linear_jac(c, cJ, P[f"layers_col.{lid}.weight"], P[f"layers_col.{lid}.bias"], mm)
        if taps is not None:
            taps[f"col{lid}_pre"] = c
        c, cJ = act(c, cJ)
        if taps is not None:
            taps[f"col{lid}_x"], taps[f"col{lid}_J"] = c, cJ
    color, colorJ = linear_jac(c, cJ, P["layer_col_out.weight"], P["layer_col_out.bias"], mm)

    # field-constraint penalties, neddf.py:259-300 (insertion order matters for the final sum)
    pen: Dict[str, Tensor] = {}
    d2 = torch.sum(aux_gg * normal, 1, keepdim=True)
    d2_rest = 3 * aux * dist_inv.detach()
    ag_scale = aux.detach() * grad_norm.detach() * distance.detach()
    pen["constraints_aux_grad"] = ag_scale * torch.square(d2 - d2_rest)
    pen["constraints_dDdt"] = torch.square(torch.relu(-1.0 + dDdt))
    pen["range_distance"] = torch.square(
        torch.relu(-4.6 - ddf_out) + torch.relu(-st.distance_range_max + ddf_out)
    )
    pen["range_aux_grad"] = torch.square(torch.relu(-4.6 - aux_out) + torch.relu(-4.6 + aux_out))
    pen["range_color"] = torch.square(torch.relu(-0.0 - color) + torch.relu(-1.0 + color)).sum(1, keepdim=True)
    pen["constraints_color"] = (colorJ * grad_d.detach().unsqueeze(2)).sum(1).square().sum(1, keepdim=True)
    total = None
    for k, v in pen.items():
        if k in cfg.penalty_weight:
            v = v * cfg.penalty_weight[k]
        total = v if total is None else total + v

    if taps is not None:
        taps.update(ddf_out=ddf_out, ddf_outJ=ddf_outJ, aux_out=aux_out, aux_outJ=aux_outJ,
                    grad_d=grad_d, aux_gg=aux_gg, dDdt=dDdt, normal=normal, colorJ=colorJ,
                    **{"pen_" + k: v for k, v in pen.items()})
    return {
        "distance": distance.view(B, S),
        "density": density.view(B, S),
        "color": color.view(B, S, 3),
        "fields_penalty": total.view(B, S),
        "aux_grad": aux.view(B, S),
    }


# --------------------------------------------------------------------------------------
# ray / sample geometry
# --------------------------------------------------------------------------------------


def make_rays(uv: Tensor, cam: CameraPose, dtype=torch.float32) -> Tuple[Tensor, Tensor]:
    """uv[B,2] pixel ids -> (ray_dir[B,3], ray_orig[B,3]).

    neddf/camera/camera.py:155-187 (+0.5 pixel centre) and
    neddf/camera/pinhole_calib.py:64-73 (unproject, RDF->RUB flip, normalise).
    """
    c = 0.5 + uv.to(dtype)
    fx, fy = torch.tensor(cam.fx, dtype=dtype), torch.tensor(cam.fy, dtype=dtype)
    x = (1.0 / fx) * (c[:, 0] - cam.cx)
    y = (1.0 / fy) * (c[:, 1] - cam.cy)
    local = torch.stack([x, -y, -torch.ones_like(x)], 1)
    local = torch.nn.functional.normalize(local, p=2, dim=1)
    R = cam.R.to(dtype)
    d = torch.matmul(R, local.T).T
    o = cam.T.to(dtype)[None, :].expand(uv.shape[0], 3)
    return d, o


def coarse_dists(rc: RenderConfig, u: Tensor) -> Tensor:
    """Stratified edges: linspace(near,far,S+1) + U*(far-near)/S (neddf/render/nerf_render.py:131-139)."""
    s1 = rc.sample_coarse + 1
    lin = torch.linspace(rc.dist_near, rc.dist_far, s1, dtype=u.dtype).reshape(1, s1)
    return lin + u * ((rc.dist_far - rc.dist_near) / rc.sample_coarse)


def point_samples(ray_dir: Tensor, ray_orig: Tensor, dists: Tensor):
    """pos = o + d*t, zero variance (neddf/ray/ray.py:88-126)."""
    pos = ray_orig.unsqueeze(1) + ray_dir.unsqueeze(1) * dists.unsqueeze(2)
    d = ray_dir.unsqueeze(1).expand_as(pos)
    return pos, d, torch.zeros_like(pos)


def cone_samples(ray_dir: Tensor, ray_orig: Tensor, dists: Tensor, ray_radius: float):
    """Conical-frustum mean / diagonal variance per edge (neddf/ray/ray.py:128-194)."""
    near = dists
    far = torch.cat([dists[:, 1:], 2 * dists[:, -1:] - dists[:, -2:-1]], 1)  # ray.py:160-163
    mu = 0.5 * (near + far)
    sg = 0.5 * (far - near)
    mu2, sg2 = mu * mu, sg * sg
    sg4 = sg2 * sg2
    m_inv = torch.reciprocal(3 * mu2 + sg2 + 1e-7)
    t_mu = mu + (2 * mu * sg2) * m_inv  # ray.py:171
    t_var = (1.0 / 3) * sg2 - (4.0 / 15) * sg4 * (12 * mu2 - sg2) * (m_inv * m_inv)  # ray.py:172-174
    r_var = ray_radius * ray_radius * ((1.0 / 4) * mu2 + (5.0 / 12) * sg2 - (4.0 / 15) * sg4 * m_inv)
    d = ray_dir.unsqueeze(1).expand(dists.shape[0], dists.shape[1], 3)
    dsq = d * d
    var = t_var[:, :, None] * dsq + r_var[:, :, None] * (1.0 - dsq)  # ray.py:185-186
    pos = ray_orig.unsqueeze(1) + d * t_mu[:, :, None]
    return pos, d, var


CONE_RAY_RADIUS = 1.0 / 1111 / math.sqrt(12)  # neddf/render/nerf_render.py:145


def make_samples(rc: RenderConfig, ray_dir, ray_orig, dists):
    if rc.sampling_type == "point":
        return point_samples(ray_dir, ray_orig, dists)
    if rc.sampling_type == "cone":
        return cone_samples(ray_dir, ray_orig, dists, CONE_RAY_RADIUS)
    raise ValueError(rc.sampling_type)


# --------------------------------------------------------------------------------------
# compositing and hierarchical resampling
# --------------------------------------------------------------------------------------


def composite(dists: Tensor, density: Tensor, color: Tensor, max_dist: float) -> Dict[str, Tensor]:
    """Alpha compositing along rays (neddf/render/base_neural_render.py:144-172).

    The last sample only supplies the far edge of the last interval.
    """
    delta = dists[:, 1:] - dists[:, :-1]
    o = 1 - torch.exp(-density[:, :-1] * delta)
    ones = torch.ones(o.shape[0], 1, dtype=o.dtype)
    t = torch.cumprod(torch.cat([ones, 1.0 - o + 1e-7], 1), 1)
    w = o * t[:, :-1]
    depth = torch.sum(w * dists[:, :-1], 1) + t[:, -1] * max_dist
    col = torch.sum(w.unsqueeze(2) * color[:, :-1, :], 1)
    return {"weight": w, "depth": depth, "color": col, "transmittance": t[:, -1]}


def integrate_penalty(dists: Tensor, penalty: Tensor) -> Tensor:
    """sum_j delta_j * penalty_j, j < S-1 (neddf/render/nerf_render.py:153-159)."""
    delta = dists[:, 1:] - dists[:, :-1]
    return torch.sum(delta.detach() * penalty[:, :-1], 1)


def sanitise_weights(weights: Tensor) -> Tensor:
    """Negative -> w*0.0, NaN -> 0 (base_neural_render.py:52-55).  The reference does this IN
    PLACE on its argument, which is the very tensor render_rays returns as "weight_coarse"."""
    w = torch.where(weights < 0.0, weights * 0.0, weights)
    return torch.where(torch.isnan(w), torch.zeros_like(w), w)


def pdf_cdf(weights: Tensor, smooth: bool = False) -> Tensor:
    """Sanitise, +1e-2, [neighbour-max smoothing when not cat_coarse, :61-68], L1-normalise, cumsum with
    leading 0 (base_neural_render.py:52-72)."""
    w = sanitise_weights(weights) + 1e-2
    if smooth and w.shape[-1] > 1:  # the reference writes weights[:, 1:-1], which is empty for one interval
        w1 = torch.maximum(w[:, 2:], w[:, 1:-1])
        w2 = torch.maximum(w[:, :-2], w[:, 1:-1])
        w = torch.cat([w[:, :1], 0.5 * (w1 + w2), w[:, -1:]], -1)
    pdf = torch.nn.functional.normalize(w, p=1.0, dim=-1)
    cdf = torch.cumsum(pdf, -1)
    return torch.cat([torch.zeros_like(cdf[..., :1]), cdf], -1)


def invert_cdf(dists: Tensor, cdf: Tensor, u: Tensor) -> Tuple[Tensor, Tensor]:
    """Inverse-CDF draw; returns (new dists [B,F], searchsorted ids int64) (base_neural_render.py:77-98)."""
    ids = torch.searchsorted(cdf, u.contiguous(), right=True)
    below = torch.clamp(ids - 1, min=0)
    above = torch.clamp(ids, max=cdf.shape[-1] - 1)
    c0, c1 = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
    d0, d1 = torch.gather(dists, 1, below), torch.gather(dists, 1, above)
    denom = c1 - c0
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)
    t = (u - c0) / denom
    return d0 + t * (d1 - d0), ids


def sample_pdf(dists: Tensor, weights: Tensor, u: Tensor, cat_coarse: bool = True) -> Tensor:
    """Hierarchical resampling (neddf/render/base_neural_render.py:27-115): with the coarse edges merged in
    (cat_coarse=True, what render_rays uses) or the new samples alone after the neighbour-max smoothing of the
    biased weights (:61-68).  ``u`` replaces the internal torch.rand."""
    cdf = pdf_cdf(weights, smooth=not cat_coarse)
    new, _ = invert_cdf(dists, cdf, u)
    merged = torch.sort(torch.cat([new, dists], -1) if cat_coarse else new, dim=-1)[0]
    if torch.any(torch.isnan(merged)):  # base_neural_render.py:105-114
        merged = torch.linspace(float(dists[0, 0]), float(dists[0, -1]), merged.shape[1],
                                dtype=dists.dtype).reshape(1, -1).expand(dists.shape[0], -1)
    return merged


# --------------------------------------------------------------------------------------
# the hot function
# --------------------------------------------------------------------------------------


def render_rays(
    P_coarse: Dict[str, Tensor],
    P_fine: Dict[str, Tensor],
    cfg: FieldConfig,
    st: FieldState,
    rc: RenderConfig,
    uv: Tensor,
    cam: CameraPose,
    u_coarse: Tensor,
    u_fine: Tensor,
    dtype=torch.float32,
    mm: Optional[MatMul] = None,
    taps: Optional[Dict[str, Tensor]] = None,
) -> Dict[str, Tensor]:
    """NeRFRender.render_rays (neddf/render/nerf_render.py:109-188).

    ``u_coarse`` [B, S_c+1] and ``u_fine`` [B, S_f+1] replace the two torch.rand draws
    (nerf_render.py:137, base_neural_render.py:75).
    """
    if dtype != torch.float32:
        P_coarse = {k: v.to(dtype) for k, v in P_coarse.items()}
        P_fine = {k: v.to(dtype) for k, v in P_fine.items()}
    ray_dir, ray_orig = make_rays(uv, cam, dtype)
    dc = coarse_dists(rc, u_coarse.to(dtype))
    pos, d, var = make_samples(rc, ray_dir, ray_orig, dc)
    vc = field_forward(P_coarse, cfg, st, pos, d, var, mm)
    ic = composite(dc, vc["density"], vc["color"], rc.max_dist)
    ic["fields_penalty"] = integrate_penalty(dc, vc["fields_penalty"])
    with torch.no_grad():
        df = sample_pdf(dc, ic["weight"].detach(), u_fine.to(dtype))
    ic["weight"] = sanitise_weights(ic["weight"])  # in-place side effect of sample_pdf, :52-55
    pos, d, var = make_samples(rc, ray_dir, ray_orig, df)
    vf = field_forward(P_fine, cfg, st, pos, d, var, mm)
    out = composite(df, vf["density"], vf["color"], rc.max_dist)
    out["fields_penalty"] = integrate_penalty(df, vf["fields_penalty"])
    for k in list(ic.keys()):
        out[k + "_coarse"] = ic[k]
    if taps is not None:
        taps.update(ray_dir=ray_dir, ray_orig=ray_orig, dists_coarse=dc, dists_fine=df,
                    density_coarse=vc["density"], color_sample_coarse=vc["color"],
                    density_fine=vf["density"], color_sample_fine=vf["color"],
                    distance_fine=vf["distance"], penalty_sample_fine=vf["fields_penalty"],
                    aux_grad_fine=vf["aux_grad"])
    return out


def image_uv(width: int, height: int, downsampling: int = 1) -> Tensor:
    """Row-major pixel grid (neddf/render/nerf_render.py:220-230)."""
    w, h = width // downsampling, height // downsampling
    us = torch.arange(w).reshape(1, w).expand(h, w).reshape(-1) * downsampling
    vs = torch.arange(h).reshape(h, 1).expand(h, w).reshape(-1) * downsampling
    return torch.stack([us, vs], 1)


def split_state_dict(sd: Dict[str, Tensor]) -> Tuple[Dict[str, Tensor], Dict[str, Tensor]]:
    """NeRFRender.state_dict() -> (coarse params, fine params) keyed like a single NeDDF."""
    pc = {k[len("network_coarse."):]: v for k, v in sd.items() if k.startswith("network_coarse.")}
    pf = {k[len("network_fine."):]: v for k, v in sd.items() if k.startswith("network_fine.")}
    return pc, pf


# --------------------------------------------------------------------------------------
# split-precision GEMM emulation (used to choose the tensor-core operand format)
# --------------------------------------------------------------------------------------


def split_matmul(fmt: str, products: int = 3) -> MatMul:
    """Emulate an error-compensated tensor-core GEMM: operands split into hi/lo parts of
    ``fmt`` ("fp16", "bf16", "tf32"), fp32 accumulate, products = 1 (hi*hi) or 3
    (hi*hi + lo*hi + hi*lo)."""

    def rnd(t: Tensor) -> Tensor:
        if fmt == "fp16":
            return t.to(torch.float16).to(torch.float32)
        if fmt == "bf16":
            return t.to(torch.bfloat16).to(torch.float32)
        if fmt == "tf32":  # round-to-nearest-even on 13 dropped bits
            i = t.contiguous().view(torch.int32)
            i = (i + 0xFFF + ((i >> 13) & 1)) & ~0x1FFF
            return i.view(torch.float32)
        raise ValueError(fmt)

    def mm(a: Tensor, b: Tensor) -> Tensor:
        ah, bh = rnd(a), rnd(b)
        out = torch.matmul(ah, bh)
        if products >= 3:
            al, bl = rnd(a - ah), rnd(b - bh)
            out = out + torch.matmul(al, bh) + torch.matmul(ah, bl)
        return out

    return mm


# --------------------------------------------------------------------------------------
# the NeRF field variant (SURVEY 8(f) item 3): same renderer, plain MLP, no Jacobian rows
# --------------------------------------------------------------------------------------


@dataclass
class NerfConfig:
    """Constructor arguments of NeRF (neddf/network/nerf.py:34-44)."""

    embed_pos_rank: int = 10
    embed_dir_rank: int = 4
    layer_count: int = 8
    layer_width: int = 256
    activation_type: str = "ReLU"
    density_activation_type: str = "ReLU"
    skips: Optional[List[int]] = None
    lowpass_alpha_offset: float = 10.0

    def __post_init__(self) -> None:
        if self.skips is None:
            self.skips = [4]

    @staticmethod
    def from_dict(d: Dict) -> "NerfConfig":
        d = {k: v for k, v in dict(d).items() if k != "_target_"}
        if d.get("skips") is not None:
            d["skips"] = [int(s) for s in d["skips"]]
        return NerfConfig(**d)

    def lowpass_alpha_at(self, it: int) -> float:
        """NeRF.set_iter (nerf.py:167-178)."""
        return float(self.embed_pos_rank) if it == -1 else self.lowpass_alpha_offset + 0.001 * it


def nerf_layer_shapes(cfg: NerfConfig) -> List[Tuple[str, int, int]]:
    """state_dict names and [in,out] shapes of the NeRF linear layers (nerf.py:86-103)."""
    in_pos, in_dir = cfg.embed_pos_rank * 6, cfg.embed_dir_rank * 6
    shapes = [("layers.0", in_pos, cfg.layer_width)]
    for lid in range(cfg.layer_count - 1):
        shapes.append((f"layers.{lid + 1}", cfg.layer_width + (in_pos if lid in cfg.skips else 0), cfg.layer_width))
    shapes.append(("outL_density", cfg.layer_width, 1))
    shapes.append(("outL_color.0", cfg.layer_width + in_dir, cfg.layer_width // 2))
    shapes.append(("outL_color.2", cfg.layer_width // 2, 3))
    return shapes


def nerf_forward(P: Dict[str, Tensor], cfg: NerfConfig, lowpass_alpha: float, pos: Tensor, dirs: Tensor,
                 var: Tensor) -> Dict[str, Tensor]:
    """NeRF.forward (neddf/network/nerf.py:107-165) on a [B,S,3] block of samples.  ``P`` holds the
    weights as [in,out] (transposed torch Linear weights) under the reference's state_dict names."""
    B, S = pos.shape[0], pos.shape[1]
    n = B * S
    x3, d3, v3 = pos.reshape(n, 3), dirs.reshape(n, 3), var.reshape(n, 3)
    E = cfg.embed_pos_rank
    scale = lowpass_scale(E, lowpass_alpha, pos.dtype).reshape(1, E, 1).expand(1, E, 3).reshape(1, 3 * E)
    scale = scale * pe_weights(v3, E)  # nerf.py:133-141
    embed_pos = pe_plain(x3, E) * torch.cat([scale, scale], 1)
    embed_dir = pe_plain(d3, cfg.embed_dir_rank)  # nerf.py:142
    act = {"ReLU": torch.relu, "LeakyReLU": torch.nn.functional.leaky_relu,
           "tanhExp": lambda t: density_act("tanhExp", t)}[cfg.activation_type]
    hx = embed_pos
    for lid in range(cfg.layer_count):  # nerf.py:144-148
        hx = act(hx @ P[f"layers.{lid}.weight"] + P[f"layers.{lid}.bias"])
        if lid in cfg.skips:
            hx = torch.cat([hx, embed_pos], 1)
    density = density_act(cfg.density_activation_type, hx @ P["outL_density.weight"] + P["outL_density.bias"])
    feat = torch.cat([hx, embed_dir], 1)  # nerf.py:151-152
    c1 = torch.relu(feat @ P["outL_color.0.weight"] + P["outL_color.0.bias"])
    color = c1 @ P["outL_color.2.weight"] + P["outL_color.2.bias"]
    return {"density": density.reshape(B, S), "color": color.reshape(B, S, 3)}


def nerf_init_params(cfg: NerfConfig, seed: int, bias_std: float = 0.05) -> Dict[str, Tensor]:
    """Seeded weights [in,out] for tests (the reference uses torch's default Linear init; goldens carry their
    weights explicitly)."""
    g = torch.Generator().manual_seed(seed)
    out: Dict[str, Tensor] = {}
    for name, cin, cout in nerf_layer_shapes(cfg):
        out[name + ".weight"] = torch.randn(cin, cout, generator=g) * math.sqrt(2.0 / (cin + cout))
        out[name + ".bias"] = torch.randn(cout, generator=g) * bias_std
    return out


# --------------------------------------------------------------------------------------
# the NeuS field variant (SURVEY 8(f) item 3): SDF trunk, one reverse-mode gradient, colour trunk
# --------------------------------------------------------------------------------------


@dataclass
class NeusConfig:
    """Constructor arguments of NeuS (neddf/network/neus.py:29-40)."""

    embed_pos_rank: int = 6
    embed_dir_rank: int = 4
    sdf_layer_count: int = 8
    sdf_layer_width: int = 256
    col_layer_count: int = 8
    col_layer_width: int = 256
    activation_type: str = "ReLU"
    init_variance: float = 0.3
    skips: Optional[List[int]] = None

    def __post_init__(self) -> None:
        if self.skips is None:
            self.skips = [4]

    @staticmethod
    def from_dict(d: Dict) -> "NeusConfig":
        d = {k: v for k, v in dict(d).items() if k != "_target_"}
        if d.get("skips") is not None:
            d["skips"] = [int(s) for s in d["skips"]]
        return NeusConfig(**d)


def neus_layer_shapes(cfg: NeusConfig) -> List[Tuple[str, int, int]]:
    """state_dict names and [in,out] shapes of the NeuS linear layers (neus.py:83-98): layers_sdf.0 .. ,
    layers_col.0 .. layers_col.{col_layer_count} (the last one is the 3-channel output)."""
    in_sdf = cfg.embed_pos_rank * 6
    in_col = 6 + cfg.embed_dir_rank * 6 + cfg.sdf_layer_width
    shapes = [("layers_sdf.0", in_sdf, cfg.sdf_layer_width)]
    for lid in range(cfg.sdf_layer_count - 1):
        shapes.append((f"layers_sdf.{lid + 1}", cfg.sdf_layer_width + (in_sdf if lid in cfg.skips else 0), cfg.sdf_layer_width))
    shapes.append(("layers_col.0", in_col, cfg.col_layer_width))
    for i in range(cfg.col_layer_count - 1):
        shapes.append((f"layers_col.{i + 1}", cfg.col_layer_width, cfg.col_layer_width))
    shapes.append((f"layers_col.{cfg.col_layer_count}", cfg.col_layer_width, 3))
    return shapes


def _neus_act(name: str) -> Callable[[Tensor], Tensor]:
    # neus.py:70-75: nn.ReLU or the plain tanhExp autograd Function (nn_module/tanh_exp.py:15-60; its backward
    # tx - x ex (tx^2 - 1), 1 above the threshold, is the derivative autograd finds for the expression below)
    return {"ReLU": torch.relu, "tanhExp": lambda t: density_act("tanhExp", t)}[name]


def neus_density(sdf: Tensor, variance: Tensor) -> Tensor:
    """neus.py:150-153, operation by operation."""
    ex = torch.exp(-variance * 10.0 * sdf)
    return variance * 10.0 * ex * torch.reciprocal(torch.square(1 + ex))


def neus_forward(P: Dict[str, Tensor], cfg: NeusConfig, pos: Tensor, dirs: Tensor) -> Dict[str, Tensor]:
    """NeuS.forward (neddf/network/neus.py:101-162) on a [B,S,3] block of samples; the normal is the reverse-mode
    gradient of the SDF with respect to the position, as in the reference (neus.py:133-142).  ``P`` holds the
    weights as [in,out] under the reference's state_dict names plus ``variance``.  Runs with autograd enabled
    whatever the caller's mode (the reference fails under no_grad: autograd.grad has nothing to differentiate)."""
    B, S = pos.shape[0], pos.shape[1]
    n = B * S
    act = _neus_act(cfg.activation_type)
    with torch.enable_grad():
        x3 = pos.detach().reshape(n, 3).clone().requires_grad_(True)
        embed_pos = pe_plain(x3, cfg.embed_pos_rank)  # neus.py:119
        embed_dir = pe_plain(dirs.reshape(n, 3), cfg.embed_dir_rank)  # neus.py:120
        hx = embed_pos
        for lid in range(cfg.sdf_layer_count):  # neus.py:122-126
            hx = act(hx @ P[f"layers_sdf.{lid}.weight"] + P[f"layers_sdf.{lid}.bias"])
            if lid in cfg.skips:
                hx = torch.cat([hx, embed_pos], 1)
        sdf = hx[:, :1]
        (gradients,) = torch.autograd.grad(sdf, x3, torch.ones_like(sdf), retain_graph=False)  # neus.py:133-142
    with torch.no_grad():
        hx = hx.detach()
        sdf = sdf.detach()
        hc = torch.cat([x3.detach(), embed_dir, gradients, hx], 1)  # neus.py:144-147
        for lid in range(cfg.col_layer_count + 1):  # every colour layer is followed by the activation, the last too
            hc = act(hc @ P[f"layers_col.{lid}.weight"] + P[f"layers_col.{lid}.bias"])
        density = neus_density(sdf, P["variance"])
    return {"sdf": sdf.reshape(B, S), "density": density.reshape(B, S), "color": hc.reshape(B, S, 3),
            "gradients": gradients.reshape(B, S, 3)}


def neus_forward_jac(P: Dict[str, Tensor], cfg: NeusConfig, pos: Tensor, dirs: Tensor) -> Dict[str, Tensor]:
    """The same network with the gradient carried FORWARD (value row + three Jacobian rows through the SDF trunk,
    the formulation of the CUDA kernel); equal to neus_forward up to rounding, checked in tests/test_neus_oracle.py."""
    B, S = pos.shape[0], pos.shape[1]
    n = B * S
    x3, d3 = pos.reshape(n, 3), dirs.reshape(n, 3)
    E = cfg.embed_pos_rank
    embed_pos, embed_J = _pe_plain_jac(x3, E)
    hidden = {"ReLU": lambda x, J: (torch.relu(x), J * (x > 0).to(x.dtype).unsqueeze(1)), "tanhExp": act_tanhexp}[cfg.activation_type]
    hx, hJ = embed_pos, embed_J
    for lid in range(cfg.sdf_layer_count):
        y, G = linear_jac(hx, hJ, P[f"layers_sdf.{lid}.weight"], P[f"layers_sdf.{lid}.bias"])
        hx, hJ = hidden(y, G)
        if lid in cfg.skips:
            hx, hJ = torch.cat([hx, embed_pos], 1), torch.cat([hJ, embed_J], 2)
    sdf, gradients = hx[:, :1], hJ[:, :, 0]
    act = _neus_act(cfg.activation_type)
    hc = torch.cat([x3, pe_plain(d3, cfg.embed_dir_rank), gradients, hx], 1)
    for lid in range(cfg.col_layer_count + 1):
        hc = act(hc @ P[f"layers_col.{lid}.weight"] + P[f"layers_col.{lid}.bias"])
    density = neus_density(sdf, P["variance"])
    return {"sdf": sdf.reshape(B, S), "density": density.reshape(B, S), "color": hc.reshape(B, S, 3),
            "gradients": gradients.reshape(B, S, 3)}


def _pe_plain_jac(x3: Tensor, embed_dim: int) -> Tuple[Tensor, Tensor]:
    """[sin p | cos p] with p[e*3+d] = 2^e x_d and its Jacobian rows J[n, i, k] = d embed_k / d x_i."""
    n = x3.shape[0]
    freq = (2.0 ** torch.arange(embed_dim, dtype=x3.dtype)).reshape(1, embed_dim, 1)
    p = (freq * x3.reshape(n, 1, 3)).reshape(n, embed_dim * 3)
    fr = freq.expand(1, embed_dim, 3).reshape(1, embed_dim * 3)
    onehot = torch.eye(3, dtype=x3.dtype).repeat(1, embed_dim).reshape(1, 3, embed_dim * 3)  # [i, e*3+d] = (d == i)
    Js = (fr * torch.cos(p)).unsqueeze(1) * onehot
    Jc = (-fr * torch.sin(p)).unsqueeze(1) * onehot
    return torch.cat([torch.sin(p), torch.cos(p)], 1), torch.cat([Js, Jc], 2)


def neus_init_params(cfg: NeusConfig, seed: int, bias_std: float = 0.05) -> Dict[str, Tensor]:
    """Seeded weights [in,out] + variance for tests (goldens carry their weights explicitly)."""
    g = torch.Generator().manual_seed(seed)
    out: Dict[str, Tensor] = {}
    for name, cin, cout in neus_layer_shapes(cfg):
        out[name + ".weight"] = torch.randn(cin, cout, generator=g) * math.sqrt(2.0 / (cin + cout))
        out[name + ".bias"] = torch.randn(cout, generator=g) * bias_std
    out["variance"] = torch.tensor(float(cfg.init_variance))
    return out


def neus_kink_distance(P: Dict[str, Tensor], cfg: NeusConfig, pos: Tensor) -> Tensor:
    """Per sample: the smallest |pre-activation| over every unit of every SDF layer.  With ReLU the normal
    (neus.py:133-142) is discontinuous where a pre-activation crosses zero, so two fp32 evaluations that differ in the
    last bit may disagree there; the parity tests use this as the witness that an outlier of the normal sits on a kink."""
    n = pos.shape[0] * pos.shape[1]
    embed_pos = pe_plain(pos.reshape(n, 3), cfg.embed_pos_rank)
    hx = embed_pos
    best = torch.full((n,), float("inf"), dtype=pos.dtype)
    for lid in range(cfg.sdf_layer_count):
        pre = hx @ P[f"layers_sdf.{lid}.weight"] + P[f"layers_sdf.{lid}.bias"]
        best = torch.minimum(best, pre.abs().min(dim=1).values)
        hx = torch.relu(pre) if cfg.activation_type == "ReLU" else density_act("tanhExp", pre)
        if lid in cfg.skips:
            hx = torch.cat([hx, embed_pos], 1)
    return best.reshape(pos.shape[0], pos.shape[1])
