"""Training restatement of the NeuS field (neddf/network/neus.py:101-162) for the tests of the training backward.

``oracle.neus_forward`` takes tanhExp in closed form, so autograd through it finds the TRUE second derivative; the
reference's tanhExp is an autograd Function that saves ex = exp(x) and tx = tanh(ex) from inside forward, without a
graph, and its backward d = tx - x ex (tx^2 - 1) is made of torch ops.  The normal is taken with
autograd.grad(create_graph=True) (neus.py:133-142), so the colour loss differentiates that backward once more - through
the explicit x only: f''_ref = ex (1 - tx^2), 0 above 20.  ``RefTanhExp`` behaves the same way, in any dtype.

Two statements of the same graph:
  neus_train_forward      the reference's structure (reverse-mode normal, create_graph=True);
  neus_train_forward_jac  the CUDA kernel's (value + three Jacobian rows carried forward, neus_train_kernel.cuh), which
                          also returns the per-layer tensors the kernel leaves behind, so that autograd can produce the
                          kernel's pre-activation gradients g_z / g_Jz as reference values.
Weights are [in,out] under the reference's state_dict names plus ``variance`` (the layout of oracle.neus_forward)."""
from typing import Dict

import numpy as np
import torch
from torch import Tensor

from oracle import neddf_oracle as orc


class RefTanhExp(torch.autograd.Function):
    """tanhExp with the reference Function's graph (nn_module/tanh_exp.py): ex, tx are constants of the backward."""

    @staticmethod
    def forward(ctx, x):
        ex = torch.exp(x)
        tx = torch.tanh(ex)
        y = x * tx
        y[x > 20.0] = x[x > 20.0]
        ctx.save_for_backward(x, ex, tx)
        return y

    @staticmethod
    def backward(ctx, g):
        x, ex, tx = ctx.saved_tensors
        d = tx - x * ex * (tx ** 2 - 1)
        d[x > 20.0] = 1.0
        return d * g


def ref_tanhexp_d2(x: Tensor) -> Tensor:
    """The second derivative double backward finds through RefTanhExp / the reference's tanhExp."""
    ex = torch.exp(x)
    tx = torch.tanh(ex)
    return torch.where(x > 20.0, torch.zeros_like(x), ex * (1 - tx * tx))


def _act(name: str):
    return {"ReLU": torch.relu, "tanhExp": RefTanhExp.apply}[name]


def neus_train_forward(P: Dict[str, Tensor], cfg: orc.NeusConfig, pos: Tensor, dirs: Tensor) -> Dict[str, Tensor]:
    """NeuS.forward as the reference builds its graph; differentiable with respect to P (and create_graph through the
    normal).  Returns sdf, density [B,S], color, normal [B,S,3]."""
    B, S = pos.shape[0], pos.shape[1]
    n = B * S
    act = _act(cfg.activation_type)
    x3 = pos.detach().reshape(n, 3).clone().requires_grad_(True)
    embed_pos = orc.pe_plain(x3, cfg.embed_pos_rank)
    embed_dir = orc.pe_plain(dirs.reshape(n, 3), cfg.embed_dir_rank)
    hx = embed_pos
    for lid in range(cfg.sdf_layer_count):
        hx = act(hx @ P[f"layers_sdf.{lid}.weight"] + P[f"layers_sdf.{lid}.bias"])
        if lid in cfg.skips:
            hx = torch.cat([hx, embed_pos], 1)
    sdf = hx[:, :1]
    (normal,) = torch.autograd.grad(sdf, x3, torch.ones_like(sdf), create_graph=True, retain_graph=True)
    hc = torch.cat([x3.detach(), embed_dir, normal, hx], 1)
    for lid in range(cfg.col_layer_count + 1):
        hc = act(hc @ P[f"layers_col.{lid}.weight"] + P[f"layers_col.{lid}.bias"])
    density = orc.neus_density(sdf, P["variance"])
    return {"sdf": sdf.reshape(B, S), "density": density.reshape(B, S), "color": hc.reshape(B, S, 3),
            "normal": normal.reshape(B, S, 3)}


def _act_jac(name: str, z: Tensor, Jz: Tensor):
    """y = f(z), J_y = f'(z) J_z with an f' whose derivative is the reference's f'' (ReLU: 0)."""
    if name == "ReLU":
        return torch.relu(z), Jz * (z > 0).to(z.dtype).unsqueeze(1)
    ex = torch.exp(z).detach()
    tx = torch.tanh(ex)
    d = tx - z * ex * (tx * tx - 1)
    d = torch.where(z > 20.0, torch.ones_like(d), d)
    return RefTanhExp.apply(z), Jz * d.unsqueeze(1)


def neus_train_forward_jac(P: Dict[str, Tensor], cfg: orc.NeusConfig, pos: Tensor, dirs: Tensor, keep: bool = False):
    """The kernel's formulation of the same graph.  With ``keep`` also returns the per-layer tensors (all retain their
    graph): E [n,n_e], EJ [n,3,n_e], per SDF layer z / Jz [n,(3,)256] and y / Jy, per colour layer z / h [n,256], the
    colour input X0 [n,n_x] and trunk features F [n,256], the head pre-activation zh [n,3]."""
    B, S = pos.shape[0], pos.shape[1]
    n = B * S
    x3, d3 = pos.reshape(n, 3), dirs.reshape(n, 3)
    E, EJ = orc._pe_plain_jac(x3, cfg.embed_pos_rank)
    t = {"E": E, "EJ": EJ, "sdf_z": [], "sdf_Jz": [], "sdf_y": [], "sdf_Jy": [], "col_z": [], "col_h": []}
    hx, hJ = E, EJ
    for lid in range(cfg.sdf_layer_count):
        z = hx @ P[f"layers_sdf.{lid}.weight"] + P[f"layers_sdf.{lid}.bias"]
        Jz = hJ @ P[f"layers_sdf.{lid}.weight"]
        if keep:
            z.retain_grad()
            Jz.retain_grad()
        y, Jy = _act_jac(cfg.activation_type, z, Jz)
        t["sdf_z"].append(z)
        t["sdf_Jz"].append(Jz)
        t["sdf_y"].append(y)
        t["sdf_Jy"].append(Jy)
        hx, hJ = y, Jy
        if lid in cfg.skips:
            hx, hJ = torch.cat([hx, E], 1), torch.cat([hJ, EJ], 2)
    sdf, normal = hx[:, :1], hJ[:, :, 0]
    act = _act(cfg.activation_type)
    X0 = torch.cat([x3, orc.pe_plain(d3, cfg.embed_dir_rank), normal], 1)
    t["X0"], t["F"] = X0, hx
    hc = torch.cat([X0, hx], 1)
    for lid in range(cfg.col_layer_count + 1):
        z = hc @ P[f"layers_col.{lid}.weight"] + P[f"layers_col.{lid}.bias"]
        if keep:
            z.retain_grad()
        hc = act(z)
        if lid < cfg.col_layer_count:
            t["col_z"].append(z)
            t["col_h"].append(hc)
        else:
            t["zh"] = z
    density = orc.neus_density(sdf, P["variance"])
    out = {"sdf": sdf.reshape(B, S), "density": density.reshape(B, S), "color": hc.reshape(B, S, 3),
           "normal": normal.reshape(B, S, 3)}
    return (out, t) if keep else out


def params_from_torch(ws, bs, names, variance, dtype, requires_grad=True) -> Dict[str, Tensor]:
    """torch-layout weights ([out,in]) -> the [in,out] dictionary of this module, leaves that require grad."""
    P = {}
    for n, w, b in zip(names, ws, bs):
        P[n + ".weight"] = torch.as_tensor(w).t().contiguous().to(dtype).requires_grad_(requires_grad)
        P[n + ".bias"] = torch.as_tensor(b).to(dtype).requires_grad_(requires_grad)
    P["variance"] = torch.as_tensor(variance).reshape(()).to(dtype).requires_grad_(requires_grad)
    return P


def _uniform(key: int, n: int) -> np.ndarray:
    """n numbers in [0, 1) on a 2^-24 grid from splitmix64 of (key, index): plain integer arithmetic, so the same bits on
    every platform and numpy / torch version."""
    golden = 0x9E3779B97F4A7C15
    z = np.arange(n, dtype=np.uint64) + np.uint64((key * golden + golden) % 2 ** 64)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(40)).astype(np.float64) / float(1 << 24)


def seeded_state_dict(cfg: orc.NeusConfig, seed: int) -> Dict[str, np.ndarray]:
    """NeuS parameters (torch layout, the reference's state_dict names) drawn like nn.Linear's default init,
    U(-1/sqrt(fan_in), 1/sqrt(fan_in)), from _uniform - so that a fixture stores a seed instead of the weights.  As in
    make_neus_golden.py the SDF channel (channel 0 of the last SDF layer) is widened and lifted and the colour head
    scaled, so that sdf, its gradient and the density vary over the samples."""
    out: Dict[str, np.ndarray] = {}
    for i, (name, cin, cout) in enumerate(orc.neus_layer_shapes(cfg)):
        bound = 1.0 / np.sqrt(float(cin))
        out[name + ".weight"] = ((2.0 * _uniform(seed * 4096 + 2 * i, cout * cin) - 1.0) * bound).astype(np.float32).reshape(cout, cin)
        out[name + ".bias"] = ((2.0 * _uniform(seed * 4096 + 2 * i + 1, cout) - 1.0) * bound).astype(np.float32)
    last, head = f"layers_sdf.{cfg.sdf_layer_count - 1}", f"layers_col.{cfg.col_layer_count}"
    out[last + ".weight"][0] *= np.float32(6.0)
    out[last + ".bias"][0] += np.float32(0.35)
    out[head + ".weight"] *= np.float32(3.0)
    out[head + ".bias"] += np.float32(0.3)
    out["variance"] = np.array(cfg.init_variance, np.float32)
    return out


def fixture_sample(g):
    """The part of a parameter gradient a fixture keeps: every 16th output row and every 4th input column of the big
    matrices, all of the 3-channel head, of the biases and of variance."""
    g = np.asarray(g)
    return g[::16, ::4] if (g.ndim == 2 and g.shape[0] > 3) else g
