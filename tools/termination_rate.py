"""Early ray termination on the NeRF and NeuS variants: one image per transmittance_eps through NeRFRender.render_image.

There are no trained NeRF / NeuS checkpoints in the repository, so each variant renders with the weights of its ReLU
golden (tests/golden/case_nerf_relu.npz, case_neus_relu.npz: the reference's networks after its own initialisation,
64 + 128 samples, cone sampling, one shared network) at the golden's 800 x 800 camera, downsampled.  For every eps:
ms per frame (CUDA events, median of the repeats after one warm-up render), executed / nominal fine evaluations
(termination_stats) and max |delta| of colour, depth and transmittance against the eps = 0 render.  Needs a GPU.

    python tools/termination_rate.py [--downsample 4] [--segments 4] [--repeats 3]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import neddf_b200  # noqa: E402

DEV = torch.device("cuda:0")
KEYS = ["color", "depth", "transmittance"]
EPS = [0.0, 1e-4, 1e-3, 1e-2]


def golden_render(variant: str):
    z = np.load(os.path.join(ROOT, "tests", "golden", f"case_{variant}_relu.npz"), allow_pickle=False)
    meta = json.loads(str(z["cfg"]))
    render = neddf_b200.NeRFRender(network_config=dict(meta["net"]), **meta["render"])
    first = "layers.0.weight" if variant == "nerf" else "layers_sdf.0.weight"
    sd = {}
    for tag in ("fine", "coarse"):
        pre = f"w_{tag}." if f"w_{tag}.{first}" in z.files else "w_fine."
        sd.update({f"network_{tag}." + k[len(pre):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(pre)})
    render.load_state_dict(sd)
    render.to(DEV)
    render.set_iter(int(z["iter"]) if "iter" in z.files else -1)
    cam = neddf_b200.Camera.from_matrix(neddf_b200.PinholeCalib(z["cam_calib"]), z["cam_R"], z["cam_T"]).to(DEV)
    cam.update_transform()
    return render, cam


def frame(render, cam, u, ds, eps, segments, repeats):
    render.transmittance_eps, render.termination_segments = eps, segments
    out = render.render_image(800, 800, cam, KEYS, ds, uniforms=u)  # warm-up (module load, handle packing)
    render.termination_stats()
    times = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = render.render_image(800, 800, cam, KEYS, ds, uniforms=u)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    st = render.termination_stats()
    return out, float(np.median(times)), {k: v // repeats for k, v in st.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--downsample", type=int, default=4)
    ap.add_argument("--segments", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("device:", q.stdout.strip() or torch.cuda.get_device_name(DEV))
    side = 800 // args.downsample
    for variant in ("nerf", "neus"):
        render, cam = golden_render(variant)
        n_pix = side * side
        g = torch.Generator().manual_seed(0)
        u = (torch.rand(n_pix, render.sample_coarse + 1, generator=g).to(DEV),
             torch.rand(n_pix, render.sample_fine + 1, generator=g).to(DEV))
        print(f"\n{variant} (weights of case_{variant}_relu.npz), {side} x {side} pixels, {render.sample_coarse} + "
              f"{render.sample_fine} samples, {args.segments} segments")
        base = None
        with torch.no_grad():
            for eps in EPS:
                out, ms, st = frame(render, cam, u, args.downsample, eps, args.segments, args.repeats)
                if base is None:
                    base = out
                    st = {"executed": n_pix * (render.sample_coarse + render.sample_fine + 2)}
                    st["nominal"] = st["executed"]
                d = {k: float((out[k] - base[k]).abs().max()) for k in KEYS}
                print(f"  eps {eps:<7g} {ms:9.1f} ms/frame  fine evaluations {st['executed']:>10d} / {st['nominal']:<10d} "
                      f"({st['executed'] / st['nominal']:.3f})  max|d| colour {d['color']:.2e} depth {d['depth']:.2e} "
                      f"transmittance {d['transmittance']:.2e}")
        render.check_status()


if __name__ == "__main__":
    main()
