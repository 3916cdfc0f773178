"""NeuS variant, training step time (csrc/neus_train.cu + neddf_wgrad; opt-in path, DESIGN 4.8): one step of the reference's
NeuS training run - render_rays of 1024 rays through NeRFRender (config/network/neus.yaml, config/render/nerf_render.yaml:
64 + 128 point samples, separate coarse network), the objective of config/loss/nerf_loss.yaml, backward - timed with CUDA
events after warm-up, with the time per kernel family from torch.profiler in a separate window, and the card's name and
power limit read in the same run.  Usage: python tools/neus_train_rate.py [n_rays] [steps]"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import neddf_b200  # noqa: E402

dev = torch.device("cuda:0")
n_rays = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
torch.manual_seed(0)
net_cfg = {"_target_": "neddf.network.NeuS", "embed_pos_rank": 6, "embed_dir_rank": 4, "sdf_layer_count": 8, "sdf_layer_width": 256,
           "col_layer_count": 8, "col_layer_width": 256, "init_variance": 0.3, "activation_type": "ReLU", "skips": [4]}
render = neddf_b200.NeRFRender(network_config=net_cfg, sample_coarse=64, sample_fine=128, dist_near=2.0, dist_far=6.0, max_dist=6.0,
                               use_coarse_network=True, sampling_type="point").to(dev)
render.set_iter(0)
for net in (render.network_coarse, render.network_fine):
    net.training_kernels = True
cam = neddf_b200.Camera.from_matrix(neddf_b200.PinholeCalib([1111.1, 1111.1, 400.0, 400.0]),
                                    torch.eye(3).numpy(), [0.0, 0.0, 4.0]).to(dev)
cam.update_transform()
g = torch.Generator().manual_seed(1)
uv = torch.stack([torch.randint(0, 800, (n_rays,), generator=g), torch.randint(0, 800, (n_rays,), generator=g)], 1).to(dev)
tc = torch.rand(n_rays, 3, generator=g).to(dev)
tm = (torch.rand(n_rays, generator=g) > 0.5).float().to(dev)


def step():
    render.zero_grad(set_to_none=True)
    out = render.render_rays(uv, cam)
    loss = 0.0
    for suffix, wc, wm in (("", 1.0, 0.05), ("_coarse", 0.1, 0.005)):  # nerf_loss.yaml, nerf_trainer.py:118-121
        loss = loss + wc * torch.mean(torch.square(out["color" + suffix] - tc))
        m = torch.clamp(1.0 - out["transmittance" + suffix], 1e-6, 1.0 - 1e-6)
        loss = loss + wm * -torch.mean(tm * torch.log(m) + (1.0 - tm) * torch.log(1.0 - m))
    loss.backward()
    return loss


for _ in range(2):  # warm-up: module load, allocator
    step()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(steps):
    loss = step()
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / steps
peak = torch.cuda.max_memory_allocated(dev) / 2 ** 30

from torch.profiler import ProfilerActivity, profile  # noqa: E402

with profile(activities=[ProfilerActivity.CUDA]) as prof:
    step()
    torch.cuda.synchronize()
fam = {}
for ev in prof.key_averages():
    if ev.device_type.name != "CUDA":
        continue
    name = ev.key
    key = next((k for k in ("neus_train_kernel", "neus_forward_kernel", "wgrad_gemm_kernel", "col_absmax_kernel", "reduce_partials",
                            "colsum_rows", "composite", "sample_pdf", "pack") if k in name), "other")
    fam[key] = fam.get(key, 0.0) + ev.device_time_total / 1e3
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print(f"card: {card}")
print(f"NeuS training step, {n_rays} rays (64 + 128 point samples, separate coarse network): {ms:.1f} ms per step "
      f"(loss {float(loss.detach()):.4f}, peak allocated {peak:.1f} GiB)")
for k, v in sorted(fam.items(), key=lambda kv: -kv[1]):
    print(f"  {k:22s} {v:9.2f} ms per step")
