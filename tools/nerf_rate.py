"""Throughput of the NeRF variant's kernels: fused-ray forward on a slice of the bench frame, on engine "fp32"
(csrc/nerf_simt.cu, tile program csrc/nerf_kernel.cuh), "tc" (csrc/nerf_tc.cu) or both.  With "both" the two engines
run alternately in one process on the same rays, and the max normalised |difference| of density and colour between
them is printed.  --frame also times NeRFRender.render_image of an 800 x 800 frame with the case_nerf_relu weights
(64 + 128 cone samples) on each engine and compares the images.  The card's name and power limit are read in the same
run.  FLOP per evaluation = 2 x sum of in x out over the linear layers (padding not counted).

    python tools/nerf_rate.py [n_rays] [fp32|tc|both] [--frame]"""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import neddf_b200
from oracle import neddf_oracle as orc  # shapes only (tools may use the oracle's config helpers)

args = [a for a in sys.argv[1:] if not a.startswith("--")]
n_rays = int(args[0]) if len(args) > 0 else 65536
which = args[1] if len(args) > 1 else "both"
engines = ("fp32", "tc") if which == "both" else (which,)
dev = torch.device("cuda:0")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip().splitlines()
print("card:", card[0] if card else torch.cuda.get_device_name(0))
torch.manual_seed(0)
net = neddf_b200.NeRF().to(dev)
net.set_iter(-1)
flop = 2 * sum(i * o for _, i, o in orc.nerf_layer_shapes(orc.NerfConfig()))
g = torch.Generator().manual_seed(0)
d = torch.nn.functional.normalize(torch.randn(n_rays, 3, generator=g), dim=-1).to(dev)
o = (torch.randn(n_rays, 3, generator=g) * 0.1).to(dev)
dists = (2.0 + 4.0 * torch.rand(n_rays, 65, generator=g).sort(dim=1).values).to(dev)
ev = n_rays * 65
reps, rounds = 3, 3
best, outs = {e: float("inf") for e in engines}, {}
with torch.no_grad():
    for e in engines:  # warm-up: handles, packing, first launch
        net.engine = e
        outs[e] = net.forward_rays(d, o, dists, "cone", neddf_b200.CONE_RAY_RADIUS)
    net.check_engine_status()
    for _ in range(rounds):  # alternate the engines so that clocks and temperature drift hit both alike
        for e in engines:
            net.engine = e
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                net.forward_rays(d, o, dists, "cone", neddf_b200.CONE_RAY_RADIUS)
            e1.record(); torch.cuda.synchronize()
            best[e] = min(best[e], e0.elapsed_time(e1) / reps)
    net.check_engine_status()
for e in engines:
    ms = best[e]
    print(f"NeRF kernel [{e}]: {ev / ms * 1e3:.3e} evaluations/s, {ev * flop / ms * 1e-9:.1f} TFLOP/s "
          f"({flop} FLOP/evaluation, {ms:.2f} ms for {ev} evaluations, best of {rounds} x {reps})")
if len(engines) == 2:
    for k in ("density", "color"):
        a, b = outs["tc"][k].double(), outs["fp32"][k].double()
        print(f"tc vs fp32 {k}: max |diff| / max |fp32| = {float((a - b).abs().max() / b.abs().max()):.3e}")

if "--frame" in sys.argv:
    from tests.test_nerf_gpu import build
    from tests.test_nerf_oracle import NerfCase
    render, cam = build(NerfCase("relu"))
    render.sample_coarse, render.sample_fine, render.sampling_type = 64, 128, "cone"
    render.set_iter(-1)
    keys = ["color", "depth", "transmittance"]
    img, t_best = {}, {e: float("inf") for e in engines}
    for e in engines:
        render.set_engine(e)
        torch.manual_seed(0)  # the same uniforms, hence the same samples, on both engines
        img[e] = render.render_image(800, 800, cam, keys, 1)
    for _ in range(2):
        for e in engines:
            render.set_engine(e)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            render.render_image(800, 800, cam, keys, 1)
            e1.record(); torch.cuda.synchronize()
            t_best[e] = min(t_best[e], e0.elapsed_time(e1))
    for e in engines:
        print(f"render_image 800x800, 64 + 128 cone samples [{e}]: {t_best[e]:.1f} ms (best of 2 after a warm-up frame)")
    if len(engines) == 2:
        for k in keys:
            a, b = img["tc"][k].double(), img["fp32"][k].double()
            print(f"frame tc vs fp32 {k}: max |diff| / max |fp32| = {float((a - b).abs().max() / b.abs().max()):.3e}")
