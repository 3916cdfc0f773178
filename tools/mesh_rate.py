"""Mesh extraction timing: the device grid evaluation (BaseNeuralField._grid_volume, what voxelize and extract_mesh
run), the marching-cubes launches (neddf_mc_count, neddf_mc_emit), the vertex-normal launch (neddf_mc_normals) and
the colour pass of extract_mesh(..., with_color=True) timed separately with CUDA events after a warm-up, with the
card's name and power limit read in the same run.

Usage: python tools/mesh_rate.py [resolution=256] [network=bunny|nerf|neus] [lipschitz]
  bunny  the bunny_smoke checkpoint (NeDDF), `distance` at 0.0275
  nerf   the seeded NeRF golden (case_nerf_relu), `density` at the volume's median
  neus   the seeded NeuS golden (case_neus_relu), `sdf` at the volume's median (the median of a 64^3 grid with a band)

With `lipschitz` the narrow band of extract_mesh(..., lipschitz=L) is timed instead (resolution up to 2048): the
coarse pass over the brick corners, the brick selection (neddf_mcb_bricks), the fine pass over the active bricks,
count + emit, normals and the colour pass, with the coarse and fine evaluation counts against n^3 and the active
bricks.
"""
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import neddf_b200  # noqa: E402
from neddf_b200 import _lib as L  # noqa: E402

res = int(sys.argv[1]) if len(sys.argv) > 1 else 256
which = sys.argv[2] if len(sys.argv) > 2 else "bunny"
dev = torch.device("cuda:0")
if which == "bunny":
    from tests.helpers import Case
    c = Case("bunny")
    render = neddf_b200.NeRFRender(network_config=c.net_cfg, **{k: v for k, v in c.render_cfg.items() if k != "_target_"})
    render.load_state_dict(c.state_dict())
    render.to(dev)
    field, thr = "distance", 0.0275
elif which == "nerf":
    from tests.test_nerf_gpu import build
    from tests.test_nerf_oracle import NerfCase
    render, field, thr = build(NerfCase("relu"))[0], "density", None
else:
    from tests.test_neus_gpu import build
    from tests.test_neus_oracle import NeusCase
    render, field, thr = build(NeusCase("relu"))[0], "sdf", None
net = render.get_network()
chunk = 1 << 20
lipschitz = float(sys.argv[3]) if len(sys.argv) > 3 else None


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1) / reps




def card_name():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def band_rate():
    """The steps of neddf_b200.mesh.narrow_band_marching_cubes on extract_mesh's grid closure, each timed."""
    import math

    from neddf_b200.mesh import _BRICK_POINTS, BRICK
    global thr
    if thr is None:
        thr = float(net._grid_volume(field, 1.1, 64, chunk).median())
    n = res
    h = 2.2 / (n - 1)
    band = float(torch.tensor(lipschitz * math.sqrt(3.0) * BRICK * h, dtype=torch.float32))
    nb = (n - 1 + BRICK - 1) // BRICK
    lib = L.lib()
    stream = L.stream_ptr(dev)
    ids = net._grid_ids(1.1, n)

    def values(active, total):
        out = torch.empty(total, dtype=torch.float32, device=dev)
        for first in range(0, total, chunk):
            m = min(chunk, total - first)
            idx = torch.empty(m, 3, dtype=torch.int32, device=dev)
            L.check(lib.neddf_mcb_points(L.ptr(active), n, first, m, L.ptr(idx), stream), "mcb_points")
            out[first:first + m] = torch.cat([net._grid_values(field, ids, idx[i:i + 65536])
                                              for i in range(0, m, 65536)])
        return out

    with torch.no_grad():
        corners, ms_coarse = timed(lambda: values(None, (nb + 1) ** 3), 2)
        ws = torch.empty(L.check(lib.neddf_mcb_bricks_workspace_bytes(n)), dtype=torch.uint8, device=dev)
        slot = torch.empty(nb ** 3, dtype=torch.int32, device=dev)
        active = torch.empty(nb ** 3, dtype=torch.int32, device=dev)
        count = torch.empty(1, dtype=torch.int64, device=dev)

        def bricks():
            L.check(lib.neddf_mcb_bricks(L.ptr(corners), n, C.c_float(thr), C.c_float(band), L.ptr(ws), L.ptr(slot),
                                         L.ptr(active), L.ptr(count), stream), "mcb_bricks")

        _, ms_bricks = timed(bricks, 10)
        n_active = int(count.item())
        fine, ms_fine = timed(lambda: values(active, n_active * _BRICK_POINTS), 2)
        cws = torch.empty(L.check(lib.neddf_mcb_workspace_bytes(n, n_active)), dtype=torch.uint8, device=dev)
        totals = torch.empty(2, dtype=torch.int64, device=dev)

        def count_kernels():
            L.check(lib.neddf_mcb_count(L.ptr(fine), n, C.c_float(thr), L.ptr(slot), L.ptr(active), n_active,
                                        L.ptr(cws), L.ptr(totals), stream), "mcb_count")

        _, ms_count = timed(count_kernels, 10)
        n_vert, n_face = totals.tolist()
        ews = torch.empty(L.check(lib.neddf_mcb_emit_workspace_bytes(n_vert, n_face)), dtype=torch.uint8, device=dev)
        verts = torch.empty(max(n_vert, 1), 3, device=dev)
        faces = torch.empty(max(n_face, 1), 3, dtype=torch.int64, device=dev)
        normals = torch.empty(max(n_vert, 1), 3, device=dev)

        def emit():
            L.check(lib.neddf_mcb_emit(L.ptr(fine), n, C.c_float(thr), L.ptr(slot), L.ptr(active), n_active,
                                       L.ptr(cws), n_vert, n_face, L.ptr(ews), L.ptr(verts), L.ptr(faces), stream),
                    "mcb_emit")

        def vertex_normals():
            L.check(lib.neddf_mcb_normals(L.ptr(fine), n, L.ptr(slot), L.ptr(active), n_active, L.ptr(cws), n_vert,
                                          n_face, L.ptr(ews), L.ptr(verts), L.ptr(faces), L.ptr(normals), stream),
                    "mcb_normals")

        _, ms_emit = timed(emit, 10)
        _, ms_normals = timed(vertex_normals, 10)
        sign = net._MESH_VIEW_SIGN.get(field)
        v64 = verts[:n_vert].double()
        world = torch.stack([-1.1 + v64[:, 2] * h, -1.1 + v64[:, 0] * h, -1.1 + v64[:, 1] * h], 1).float()
        view = normals[:n_vert][:, [2, 0, 1]] * sign
        _, ms_color = timed(lambda: net._vertex_colors(world, view), 10)
    n_coarse, n_fine = (nb + 1) ** 3, n_active * _BRICK_POINTS
    total = ms_coarse + ms_bricks + ms_fine + ms_count + ms_emit + ms_normals + ms_color
    print(f"card: {card_name()}")
    print(f"{which} {field} at {thr:g}, {n}^3 grid, narrow band L = {lipschitz:g} (band {band:.6g}): {n_vert} vertices, "
          f"{n_face} faces")
    print(f"evaluations: coarse {n_coarse} ({n_coarse / n ** 3:.3%} of n^3) + fine {n_fine} ({n_fine / n ** 3:.3%}) "
          f"= {(n_coarse + n_fine) / n ** 3:.3%}; active bricks {n_active} of {nb ** 3} ({n_active / nb ** 3:.3%})")
    print(f"engine {getattr(net, 'engine', '-')}: coarse pass {ms_coarse:.1f} ms, bricks {ms_bricks:.3f} ms, "
          f"fine pass {ms_fine:.1f} ms, count {ms_count:.2f} ms + emit {ms_emit:.2f} ms, normals {ms_normals:.3f} ms, "
          f"colour {ms_color:.3f} ms; total {total:.1f} ms")
    print(f"workspace: bricks {ws.numel() / 2 ** 20:.0f} MiB, count {cws.numel() / 2 ** 20:.0f} MiB, "
          f"emit {ews.numel() / 2 ** 20:.0f} MiB")


if lipschitz is not None:
    band_rate()
    sys.exit(0)
vol, ms_grid = timed(lambda: net._grid_volume(field, 1.1, res, chunk), 2)
if thr is None:
    thr = float(vol.median())
n0 = n1 = n2 = res
lib = L.lib()
stream = L.stream_ptr(dev)
ws = torch.empty(L.check(lib.neddf_mc_workspace_bytes(n0, n1, n2)), dtype=torch.uint8, device=dev)
totals = torch.empty(2, dtype=torch.int64, device=dev)


def count():
    L.check(lib.neddf_mc_count(L.ptr(vol), n0, n1, n2, C.c_float(thr), L.ptr(ws), L.ptr(totals), stream), "mc_count")


_, ms_count = timed(count, 10)
n_vert, n_face = totals.tolist()
verts = torch.empty(max(n_vert, 1), 3, device=dev)
faces = torch.empty(max(n_face, 1), 3, dtype=torch.int64, device=dev)


def emit():
    L.check(lib.neddf_mc_emit(L.ptr(vol), n0, n1, n2, C.c_float(thr), L.ptr(ws), L.ptr(verts), L.ptr(faces), stream),
            "mc_emit")


_, ms_emit = timed(emit, 10)
normals = torch.empty(max(n_vert, 1), 3, device=dev)


def vertex_normals():
    L.check(lib.neddf_mc_normals(L.ptr(vol), n0, n1, n2, C.c_float(thr), L.ptr(ws), L.ptr(verts), L.ptr(faces),
                                 L.ptr(normals), stream), "mc_normals")


_, ms_normals = timed(vertex_normals, 10)
# the colour pass of extract_mesh(..., with_color=True): world positions, view direction against the normal
sign = net._MESH_VIEW_SIGN.get(field)
ms_color = None
if sign is not None and n_vert:
    h = 2.2 / (res - 1)
    v64 = verts[:n_vert].double()
    world = torch.stack([-1.1 + v64[:, 2] * h, -1.1 + v64[:, 0] * h, -1.1 + v64[:, 1] * h], 1).float()
    view = normals[:n_vert][:, [2, 0, 1]] * sign
    _, ms_color = timed(lambda: net._vertex_colors(world, view), 10)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print(f"card: {card}")
print(f"{which} {field} at {thr:g}, {res}^3 grid: {n_vert} vertices, {n_face} faces, workspace {ws.numel() / 2 ** 20:.0f} MiB")
print(f"grid evaluation ({net.__class__.__name__}, engine {getattr(net, 'engine', '-')}): {ms_grid:.1f} ms, "
      f"{res ** 3 / ms_grid * 1e3:.3e} points/s")
print(f"marching cubes: count {ms_count:.2f} ms + emit {ms_emit:.2f} ms = {ms_count + ms_emit:.2f} ms, "
      f"{(res - 1) ** 3 / (ms_count + ms_emit) * 1e3:.3e} cubes/s")
print(f"vertex normals: {ms_normals:.3f} ms")
print(f"colour pass: {ms_color:.3f} ms ({n_vert} vertices)" if ms_color is not None else
      f"colour pass: {field} has no outside, not run")
