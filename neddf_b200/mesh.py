"""Triangle meshes from a field: marching cubes on the GPU (csrc/mcubes.cu, narrow band csrc/mcubes_band.cu) and a
binary PLY writer.

The reference meshes a trained field in its Open3D visualiser (scripts/fields_visualizer.py:528-567): ``voxelize``
of the distance field, PyMCubes at threshold 0.0275, a ``.dae`` file.  Here the grid, its evaluation and the
marching cubes stay on the device, and ``python -m neddf_b200.mesh RUN_DIR`` is the headless equivalent:

    python -m neddf_b200.mesh outputs/bunny_smoke [--epoch 2000] [--resolution 64] [--threshold T] [--field NAME]
                              [--out PATH] [--color] [--lipschitz L]

It reads ``RUN_DIR/.hydra/config.yaml``, loads ``RUN_DIR/models/model_{epoch:05}.pth`` into a NeRFRender, meshes
``get_network()`` with ``extract_mesh`` and writes ``RUN_DIR/mesh/mesh_{resolution}_threshold{threshold}.ply``.
Defaults per network: NeDDF ``distance`` at 0.0275 (the visualiser's), NeuS ``sdf`` at 0.0; NeRF has no canonical
level and needs ``--threshold`` (of its ``density`` field).  ``--color`` adds per-vertex normals and the field's
colour at every vertex to the PLY (``extract_mesh(..., with_color=True)``).

The dense grid stops at 512 points per axis.  ``--lipschitz L`` (NeDDF ``distance``, NeuS ``sdf``) evaluates the field
only in bricks of 8^3 cells whose corners lie within ``L * sqrt(3) * 8 * h`` of the level
(``narrow_band_marching_cubes``), which reaches 2048 and equals the dense mesh wherever the field is L-Lipschitz:

    python -m neddf_b200.mesh outputs/bunny_smoke --resolution 1024 --lipschitz 1.0 [--color]
"""
import argparse
import math
import os
import sys
from typing import Optional

import numpy as np
import torch
from torch import Tensor

from . import _lib as L

MAX_DIM = 512


def marching_cubes(volume: Tensor, threshold: float, normals: bool = False):
    """Mesh the level set ``volume == threshold`` of a contiguous fp32 CUDA volume [n0, n1, n2] (each dimension in
    [2, 512]).  Returns (vertices [V,3] fp32, faces [F,3] int64) on the volume's device; ``normals=True`` adds the
    unit vertex normals [V,3] fp32 (and leaves vertices and faces bit for bit as they are without it).

    Index space, PyMCubes' convention: vertex (i, j, k) addresses ``volume[i, j, k]``.  A corner is inside iff
    ``v < threshold``; a cube with a non-finite corner emits nothing.  The face-consistent case table makes a closed
    level set a closed, edge-manifold mesh; the normal ``(v1 - v0) x (v2 - v0)`` points toward increasing value
    (outward for a distance or SDF, inward for a density).  A vertex normal is the normalised sum of the unnormalised
    normals of its faces (area weighted), summed in face order with every step rounded on its own; where that sum has
    zero length it is the vertex's edge axis, signed toward increasing value.  The output order is deterministic.
    Exactly one host synchronisation, to read the vertex and face counts."""
    if not isinstance(volume, torch.Tensor):
        raise TypeError("marching_cubes: volume must be a torch.Tensor")
    if not volume.is_cuda:
        raise ValueError("marching_cubes: volume must be a CUDA tensor (the kernels have no CPU implementation)")
    if volume.dtype != torch.float32:
        raise ValueError(f"marching_cubes: volume must be float32, got {volume.dtype}")
    if volume.dim() != 3:
        raise ValueError(f"marching_cubes: volume must be 3-D, got shape {tuple(volume.shape)}")
    if not volume.is_contiguous():
        raise ValueError("marching_cubes: volume must be contiguous")
    n0, n1, n2 = (int(s) for s in volume.shape)
    if min(n0, n1, n2) < 2 or max(n0, n1, n2) > MAX_DIM:
        raise ValueError(f"marching_cubes: every dimension must be in [2, {MAX_DIM}], got {(n0, n1, n2)}")
    thr = float(threshold)
    if not math.isfinite(thr) or abs(thr) > float(np.finfo(np.float32).max):
        raise ValueError(f"marching_cubes: threshold must be a finite fp32 value, got {threshold!r}")
    device = volume.device
    lib = L.lib()
    with torch.cuda.device(device):
        stream = L.stream_ptr(device)
        n_bytes = L.check(lib.neddf_mc_workspace_bytes(n0, n1, n2), "mc_workspace_bytes")
        ws = torch.empty(n_bytes, dtype=torch.uint8, device=device)
        totals = torch.empty(2, dtype=torch.int64, device=device)
        L.check(lib.neddf_mc_count(L.ptr(volume), n0, n1, n2, thr, L.ptr(ws), L.ptr(totals), stream), "mc_count")
        n_vert, n_face = (int(v) for v in totals.tolist())
        vertices = torch.empty(n_vert, 3, dtype=torch.float32, device=device)
        faces = torch.empty(n_face, 3, dtype=torch.int64, device=device)
        L.check(lib.neddf_mc_emit(L.ptr(volume), n0, n1, n2, thr, L.ptr(ws), L.ptr(vertices) if n_vert else None,
                                  L.ptr(faces) if n_face else None, stream), "mc_emit")
        if not normals:
            return vertices, faces
        vnormals = torch.empty(n_vert, 3, dtype=torch.float32, device=device)
        L.check(lib.neddf_mc_normals(L.ptr(volume), n0, n1, n2, thr, L.ptr(ws), L.ptr(vertices) if n_vert else None,
                                     L.ptr(faces) if n_face else None, L.ptr(vnormals) if n_vert else None, stream),
                "mc_normals")
    return vertices, faces, vnormals


BAND_MAX_DIM = 2048
BRICK = 8  # cells per brick and axis of the narrow band (csrc/mcubes_band.cu)
_BRICK_POINTS = (BRICK + 1) ** 3
_EVAL_CHUNK = 1 << 22  # grid points per ``evaluate`` call


def narrow_band_marching_cubes(evaluate, n: int, threshold: float, band: float, normals: bool = False):
    """Mesh the level set ``v == threshold`` of an n^3 grid (n in [2, 2048]) evaluating ``v`` only near it.

    ``evaluate(idx)`` receives int32 grid indices [m, 3] of points (i, j, k) on the current CUDA device and returns
    their fp32 values [m] on that device; it is called in chunks of at most 2^22 points.  The grid's cells are cut
    into bricks of 8^3 cells.  A first pass evaluates the (nb + 1)^3 brick corners, nb = ceil((n - 1) / 8); a brick is
    kept if a corner value is non-finite or all 8 lie within ``band`` of ``threshold`` (fp32), and a second pass
    evaluates the 9^3 points of every kept brick (``(nb + 1)^3 + 729 A`` evaluations for A kept bricks).  The kept
    bricks are meshed by the rule and case table of ``marching_cubes``.

    If the values are L-Lipschitz on the grid and ``band >= L * sqrt(3) * 8 * h`` (h the grid spacing in the units of
    ``evaluate``'s positions), every brick that holds an emitting cube is kept.  Whenever that holds, the result is
    what ``marching_cubes`` returns for the dense volume ``volume[i, j, k] = evaluate(i, j, k)``: the same vertices,
    faces and (``normals=True``) normals, in the same order, bit for bit.  Two host synchronisations: the kept
    bricks' count and the vertex and face counts."""
    if not callable(evaluate):
        raise TypeError("narrow_band_marching_cubes: evaluate must be callable")
    if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or not 2 <= n <= BAND_MAX_DIM:
        raise ValueError(f"narrow_band_marching_cubes: n must be an integer in [2, {BAND_MAX_DIM}], got {n!r}")
    n = int(n)
    thr, band = float(threshold), float(band)
    f32_max = float(np.finfo(np.float32).max)
    if not math.isfinite(thr) or abs(thr) > f32_max:
        raise ValueError(f"narrow_band_marching_cubes: threshold must be a finite fp32 value, got {threshold!r}")
    if not math.isfinite(band) or not 0.0 <= band <= f32_max:
        raise ValueError(f"narrow_band_marching_cubes: band must be a finite fp32 value >= 0, got {band!r}")
    device = torch.device("cuda", torch.cuda.current_device())
    lib = L.lib()
    stream = L.stream_ptr(device)
    nb = (n - 1 + BRICK - 1) // BRICK

    def values(active, total):
        out = torch.empty(total, dtype=torch.float32, device=device)
        for first in range(0, total, _EVAL_CHUNK):
            m = min(_EVAL_CHUNK, total - first)
            idx = torch.empty(m, 3, dtype=torch.int32, device=device)
            L.check(lib.neddf_mcb_points(L.ptr(active), n, first, m, L.ptr(idx), stream), "mcb_points")
            v = evaluate(idx)
            if not (isinstance(v, torch.Tensor) and v.dtype == torch.float32 and v.device == device
                    and v.numel() == m):
                raise ValueError(f"narrow_band_marching_cubes: evaluate must return {m} fp32 values on {device}")
            out[first:first + m] = v.reshape(-1)
        return out

    def empty():
        e = (torch.empty(0, 3, dtype=torch.float32, device=device), torch.empty(0, 3, dtype=torch.int64, device=device))
        return e + (torch.empty(0, 3, dtype=torch.float32, device=device),) if normals else e

    corners = values(None, (nb + 1) ** 3)
    ws = torch.empty(L.check(lib.neddf_mcb_bricks_workspace_bytes(n), "mcb_bricks_workspace_bytes"), dtype=torch.uint8,
                     device=device)
    slot = torch.empty(nb ** 3, dtype=torch.int32, device=device)
    active = torch.empty(nb ** 3, dtype=torch.int32, device=device)
    count = torch.empty(1, dtype=torch.int64, device=device)
    L.check(lib.neddf_mcb_bricks(L.ptr(corners), n, thr, band, L.ptr(ws), L.ptr(slot), L.ptr(active), L.ptr(count),
                                 stream), "mcb_bricks")
    n_active = int(count.item())
    if n_active == 0:
        return empty()
    fine = values(active, n_active * _BRICK_POINTS)
    ws = torch.empty(L.check(lib.neddf_mcb_workspace_bytes(n, n_active), "mcb_workspace_bytes"), dtype=torch.uint8,
                     device=device)
    totals = torch.empty(2, dtype=torch.int64, device=device)
    L.check(lib.neddf_mcb_count(L.ptr(fine), n, thr, L.ptr(slot), L.ptr(active), n_active, L.ptr(ws), L.ptr(totals),
                                stream), "mcb_count")
    n_vert, n_face = (int(v) for v in totals.tolist())
    if n_vert == 0:
        return empty()
    ews = torch.empty(L.check(lib.neddf_mcb_emit_workspace_bytes(n_vert, n_face), "mcb_emit_workspace_bytes"),
                      dtype=torch.uint8, device=device)
    vertices = torch.empty(n_vert, 3, dtype=torch.float32, device=device)
    faces = torch.empty(n_face, 3, dtype=torch.int64, device=device)
    L.check(lib.neddf_mcb_emit(L.ptr(fine), n, thr, L.ptr(slot), L.ptr(active), n_active, L.ptr(ws), n_vert, n_face,
                               L.ptr(ews), L.ptr(vertices), L.ptr(faces), stream), "mcb_emit")
    if not normals:
        return vertices, faces
    vnormals = torch.empty(n_vert, 3, dtype=torch.float32, device=device)
    L.check(lib.neddf_mcb_normals(L.ptr(fine), n, L.ptr(slot), L.ptr(active), n_active, L.ptr(ws), n_vert, n_face,
                                  L.ptr(ews), L.ptr(vertices), L.ptr(faces), L.ptr(vnormals), stream), "mcb_normals")
    return vertices, faces, vnormals


# PLY property types this module writes and reads
_PLY_TYPES = {"float": "<f4", "uchar": "u1"}
_XYZ, _NORMAL, _RGB = ("x", "y", "z"), ("nx", "ny", "nz"), ("red", "green", "blue")


def _columns(a, dtype, name: str, n: int) -> np.ndarray:
    c = np.ascontiguousarray(torch.as_tensor(a).detach().cpu().numpy(), dtype=dtype).reshape(-1, 3)
    if len(c) != n:
        raise ValueError(f"write_ply: {name} has {len(c)} rows for {n} vertices")
    return c


def write_ply(path: str, vertices, faces, normals=None, colors=None) -> None:
    """Binary little-endian PLY.  Per vertex, packed: float x, y, z; float nx, ny, nz when ``normals`` is given;
    uchar red, green, blue when ``colors`` is given.  Float colours are converted by the rule of the project's image
    writer (``eval_io.color_to_uint8``: clamp(c * 255, 0, 255), truncated); uint8 colours are written as they are.
    Per face: a ``uchar`` count and int32 indices."""
    from .eval_io import color_to_uint8
    v = np.ascontiguousarray(torch.as_tensor(vertices).detach().cpu().numpy(), dtype="<f4").reshape(-1, 3)
    f = torch.as_tensor(faces).detach().cpu().numpy().reshape(-1, 3)
    if len(f) and (f.min() < 0 or f.max() >= len(v)):
        raise ValueError("write_ply: face index out of range")
    props = [(_XYZ, "float", v)]
    if normals is not None:
        props.append((_NORMAL, "float", _columns(normals, "<f4", "normals", len(v))))
    if colors is not None:
        c = torch.as_tensor(colors).detach()
        c = c if c.dtype == torch.uint8 else color_to_uint8(c.to(torch.float32))
        props.append((_RGB, "uchar", _columns(c, "u1", "colors", len(v))))
    vrec = np.empty(len(v), dtype=[(name, _PLY_TYPES[t]) for names, t, _ in props for name in names])
    for names, _, cols in props:
        for q, name in enumerate(names):
            vrec[name] = cols[:, q]
    rec = np.empty(len(f), dtype=[("n", "u1"), ("idx", "<i4", (3,))])
    rec["n"] = 3
    rec["idx"] = f
    vprops = "".join(f"property {t} {name}\n" for names, t, _ in props for name in names)
    header = (f"ply\nformat binary_little_endian 1.0\nelement vertex {len(v)}\n{vprops}"
              f"element face {len(f)}\nproperty list uchar int vertex_indices\nend_header\n")
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(vrec.tobytes())
        fh.write(rec.tobytes())


def read_ply(path: str, attributes: bool = False):
    """Read back what ``write_ply`` writes: (vertices [V,3] float32, faces [F,3] int64).  The vertex record is
    parsed from the header.  ``attributes=True`` returns a dict instead: ``vertices``, ``faces``, and ``normals``
    [V,3] float32 / ``colors`` [V,3] uint8 when the file has them."""
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    counts, vprops, element = {}, [], None
    for line in data[:end].decode("ascii").splitlines():
        parts = line.split()
        if parts[:1] == ["format"] and parts[1] != "binary_little_endian":
            raise ValueError(f"read_ply: unsupported format {parts[1]}")
        if parts[:1] == ["element"]:
            element = parts[1]
            counts[element] = int(parts[2])
        if parts[:1] == ["property"] and element == "vertex":
            if parts[1] not in _PLY_TYPES:
                raise ValueError(f"read_ply: unsupported vertex property type {parts[1]}")
            vprops.append((parts[2], _PLY_TYPES[parts[1]]))
    nv, nf = counts["vertex"], counts["face"]
    vrec = np.frombuffer(data, dtype=vprops, count=nv, offset=end)
    rec = np.frombuffer(data, dtype=[("n", "u1"), ("idx", "<i4", (3,))], count=nf, offset=end + vrec.dtype.itemsize * nv)
    if nf and not (rec["n"] == 3).all():
        raise ValueError("read_ply: only triangle faces are supported")

    def cols(names, dtype):
        return np.stack([vrec[name] for name in names], 1).astype(dtype).reshape(nv, 3)

    v, f = cols(_XYZ, np.float32), rec["idx"].astype(np.int64)
    if not attributes:
        return v, f
    out = {"vertices": v, "faces": f}
    names = vrec.dtype.names
    if all(name in names for name in _NORMAL):
        out["normals"] = cols(_NORMAL, np.float32)
    if all(name in names for name in _RGB):
        out["colors"] = cols(_RGB, np.uint8)
    return out


def load_run(run_dir: str, epoch: int = 2000, device: str = "cuda:0"):
    """The NeRFRender of a training run: ``RUN_DIR/.hydra/config.yaml`` with ``RUN_DIR/models/model_{epoch:05}.pth``
    loaded, on ``device``."""
    import yaml

    from .render import NeRFRender

    with open(os.path.join(run_dir, ".hydra", "config.yaml")) as fh:
        cfg = yaml.safe_load(fh)
    render_cfg = {k: v for k, v in cfg["render"].items() if k != "_target_"}
    render = NeRFRender(network_config=cfg["network"], **render_cfg)
    state = torch.load(os.path.join(run_dir, "models", f"model_{epoch:05}.pth"), map_location="cpu")
    render.load_state_dict(state)
    render.to(torch.device(device))
    return render


def mesh_run(run_dir: str, epoch: int = 2000, resolution: int = 64, threshold: Optional[float] = None,
             field: Optional[str] = None, out: Optional[str] = None, cube_range: float = 1.1,
             device: str = "cuda:0", color: bool = False, lipschitz: Optional[float] = None) -> str:
    """The headless half of the reference visualiser's main / generate_mesh: returns the written PLY's path.
    ``color=True`` also writes the vertex normals and colours of ``extract_mesh(..., with_color=True)``;
    ``lipschitz`` meshes through the narrow band (``extract_mesh(..., lipschitz=L)``)."""
    from .network import LEVEL_DEFAULTS

    net = load_run(run_dir, epoch, device).get_network()
    default_field, default_thr = LEVEL_DEFAULTS[type(net).__name__]
    field = field or default_field
    if threshold is None:
        threshold = default_thr
    if threshold is None:
        raise ValueError(f"{type(net).__name__} has no default iso-level: pass --threshold")
    mesh = net.extract_mesh(field, threshold, cube_range=cube_range, cube_resolution=resolution, with_color=color,
                            lipschitz=lipschitz)
    if out is None:
        os.makedirs(os.path.join(run_dir, "mesh"), exist_ok=True)
        out = os.path.join(run_dir, "mesh", f"mesh_{resolution}_threshold{threshold}.ply")
    write_ply(out, *mesh)
    return out


def main(argv=None) -> None:
    p = argparse.ArgumentParser(prog="python -m neddf_b200.mesh", description=__doc__.split("\n\n")[0])
    p.add_argument("run_dir", help="training output directory holding .hydra/config.yaml and models/")
    p.add_argument("--epoch", type=int, default=2000, help="epoch number of the model file")
    p.add_argument("--resolution", type=int, default=64,
                   help=f"grid points per axis (2..{MAX_DIM}; up to {BAND_MAX_DIM} with --lipschitz)")
    p.add_argument("--threshold", type=float, default=None, help="iso-level (default: 0.0275 NeDDF, 0.0 NeuS)")
    p.add_argument("--field", default=None, help="field to mesh (default: distance NeDDF, sdf NeuS, density NeRF)")
    p.add_argument("--out", default=None, help="output PLY path (default: RUN_DIR/mesh/mesh_{res}_threshold{thr}.ply)")
    p.add_argument("--color", action="store_true",
                   help="also write vertex normals and the field's colour at every vertex (distance / sdf / density)")
    p.add_argument("--lipschitz", type=float, default=None,
                   help="a bound L on the field's gradient norm: evaluate the grid only in a narrow band around the "
                        "surface (distance NeDDF, sdf NeuS); the mesh equals the dense one wherever the bound holds")
    a = p.parse_args(argv)
    if a.resolution > MAX_DIM and a.lipschitz is None:
        p.error(f"--resolution {a.resolution} is above {MAX_DIM}: the dense grid stops there; pass --lipschitz L to "
                f"mesh through the narrow band (up to {BAND_MAX_DIM})")
    path = mesh_run(a.run_dir, a.epoch, a.resolution, a.threshold, a.field, a.out, color=a.color,
                    lipschitz=a.lipschitz)
    v, f = read_ply(path)
    print(f"wrote {path}: {len(v)} vertices, {len(f)} faces")


if __name__ == "__main__":
    sys.exit(main())
