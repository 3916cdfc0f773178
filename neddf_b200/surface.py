"""Sphere-traced surface images of a training run (``NeRFRender.render_surface``), headless:

    python -m neddf_b200.surface outputs/bunny_smoke [--epoch 2000] [--views 8] [--size 400]

It loads the run as ``python -m neddf_b200.mesh`` does (``RUN_DIR/.hydra/config.yaml`` and
``RUN_DIR/models/model_{epoch:05}.pth``), places ``views`` cameras on an orbit of radius 4.0311 around the origin,
30 degrees above the xy plane and looking at the origin (the benchmark's pose convention, same field of view), and
writes ``RUN_DIR/surface/{k:03}_{color,normal,depth}.png`` at ``size`` x ``size``.  The images use the trainer's uint8
rule (``eval_io.color_to_uint8``, arrays written as the trainer writes them): colour as it is, the normal as
(n + 1) / 2, the depth as (t - near) / (far - near), so misses are white in the depth image.
"""
import argparse
import math
import os
import sys
from typing import List

import numpy as np
import torch

ORBIT_RADIUS = 4.0311
ORBIT_ELEVATION = math.radians(30.0)
FOV_X = 0.6911112070083618  # radians, the benchmark camera's


def orbit_pose(k: int, views: int, size: int):
    """(R [3,3], T [3], calib [fx, fy, cx, cy]) of camera k of ``views`` on the orbit; columns of R are the camera's
    right, up and back axes (back points from the origin to the camera)."""
    a = 2.0 * math.pi * k / views
    back = np.array([math.cos(a) * math.cos(ORBIT_ELEVATION), math.sin(a) * math.cos(ORBIT_ELEVATION),
                     math.sin(ORBIT_ELEVATION)])
    right = np.cross([0.0, 0.0, 1.0], back)
    right /= np.linalg.norm(right)
    up = np.cross(back, right)
    R = np.stack([right, up, back], 1).astype(np.float32)
    T = (ORBIT_RADIUS * back).astype(np.float32)
    focal = 0.5 * size / math.tan(0.5 * FOV_X)
    return R, T, np.array([focal, focal, 0.5 * size, 0.5 * size], dtype=np.float32)


def surface_images(img, near: float, far: float) -> dict:
    """uint8 host images of one ``render_surface`` result: color [h,w,3], normal [h,w,3], depth [h,w]."""
    from .eval_io import color_to_uint8
    return {"color": color_to_uint8(img["color"]).cpu().numpy(),
            "normal": color_to_uint8((img["normal"] + 1.0) * 0.5).cpu().numpy(),
            "depth": color_to_uint8((img["depth"] - near) / (far - near)).cpu().numpy()[..., 0]}


def surface_run(run_dir: str, epoch: int = 2000, views: int = 8, size: int = 400, device: str = "cuda:0") -> List[str]:
    """Render ``views`` orbit views of the run's surface and write their PNGs; returns the written paths."""
    import cv2

    from . import Camera, PinholeCalib
    from .mesh import load_run

    if views < 1 or size < 1:
        raise ValueError(f"surface_run: need views >= 1 and size >= 1, got {views}, {size}")
    render = load_run(run_dir, epoch, device)
    out_dir = os.path.join(run_dir, "surface")
    os.makedirs(out_dir, exist_ok=True)
    paths = []
    for k in range(views):
        R, T, calib = orbit_pose(k, views, size)
        cam = Camera.from_matrix(PinholeCalib(calib), R, T).to(torch.device(device))
        cam.update_transform()
        img = render.render_surface(size, size, cam)
        for name, arr in surface_images(img, render.dist_near, render.dist_far).items():
            path = os.path.join(out_dir, f"{k:03}_{name}.png")
            if not cv2.imwrite(path, arr):
                raise OSError(f"surface_run: could not write {path}")
            paths.append(path)
    return paths


def main(argv=None) -> None:
    p = argparse.ArgumentParser(prog="python -m neddf_b200.surface", description=__doc__.split("\n\n")[0])
    p.add_argument("run_dir", help="training output directory holding .hydra/config.yaml and models/")
    p.add_argument("--epoch", type=int, default=2000, help="epoch number of the model file")
    p.add_argument("--views", type=int, default=8, help="cameras on the orbit")
    p.add_argument("--size", type=int, default=400, help="image width and height in pixels")
    a = p.parse_args(argv)
    paths = surface_run(a.run_dir, a.epoch, a.views, a.size)
    print(f"wrote {len(paths)} images to {os.path.dirname(paths[0])}")


if __name__ == "__main__":
    sys.exit(main())
