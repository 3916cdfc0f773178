"""Time NeRFRender.render_surface against render_image on one frame, per engine.

Usage: python tools/surface_rate.py [size=800] [reps=3]

The bunny_smoke checkpoint (NeDDF) with the benchmark camera (``bench.synthetic_pose(0)``, radius 4.0311) at
size x size, traced at the default level 0.0275 and at 0.07.  Per engine it reports the trace time, the field
evaluations per ray (the sum of ``steps`` plus 6 per hit for the central-difference normals, over all rays; the
colour pass is one more evaluation per hit, not counted), the time the host spends in the per-iteration live-count
reads, and render_image (colour and depth) of the same frame.  The card's name and power limit are printed in the same
run.
"""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import neddf_b200  # noqa: E402

size = int(sys.argv[1]) if len(sys.argv) > 1 else 800
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
dev = torch.device("cuda:0")

from bench import synthetic_pose  # noqa: E402
from tests.helpers import Case  # noqa: E402

c = Case("bunny")
render = neddf_b200.NeRFRender(network_config=c.net_cfg, **{k: v for k, v in c.render_cfg.items() if k != "_target_"})
render.load_state_dict(c.state_dict())
render.to(dev)
render.set_iter(-1)
R, T, calib = synthetic_pose(0)
calib = np.array([calib[0] * size / (2 * calib[2]), calib[1] * size / (2 * calib[3]), 0.5 * size, 0.5 * size], np.float32)
cam = neddf_b200.Camera.from_matrix(neddf_b200.PinholeCalib(calib), R, T).to(dev)
cam.update_transform()
net = render.get_network()


class CountReads:
    """Wraps Tensor.item to time the host's blocking count reads inside trace_surface."""

    def __enter__(self):
        self.orig, self.ms, self.n = torch.Tensor.item, 0.0, 0
        outer = self

        def item(t):
            t0 = time.perf_counter()
            v = outer.orig(t)
            outer.ms += 1e3 * (time.perf_counter() - t0)
            outer.n += 1
            return v
        torch.Tensor.item = item
        return self

    def __exit__(self, *a):
        torch.Tensor.item = self.orig


def timed(fn):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    return out, 1e3 * (time.perf_counter() - t0) / reps


card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(f"card: {card}")
print(f"frame {size}x{size} ({size * size} rays), bench camera, bunny_smoke checkpoint, {reps} timed reps")
for engine in ("fp32", "tc", "tc2"):
    render.set_engine(engine)
    _, ms_img = timed(lambda: render.render_image(size, size, cam, ["color", "depth"]))
    for level in (None, 0.07):
        img, ms = timed(lambda: render.render_surface(size, size, cam, level=level))
        with CountReads() as cr:
            torch.cuda.synchronize()
            render.render_surface(size, size, cam, level=level)
            torch.cuda.synchronize()
        hits = int(img["hit"].sum())
        evals = int(img["steps"].sum()) + 6 * hits
        print(f"{engine:5s} level {net.surface_level(level):.4f}: trace {ms:8.1f} ms, hits {hits:6d}, "
              f"evaluations/ray {evals / (size * size):6.2f} (max steps {int(img['steps'].max())}), "
              f"count reads {cr.n} taking {cr.ms:6.1f} ms ({100 * cr.ms / ms:4.1f} % of the trace, includes waiting "
              f"for the preceding launches), render_image {ms_img:8.1f} ms, ratio {ms_img / ms:6.1f}x")
