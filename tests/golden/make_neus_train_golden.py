#!/usr/bin/env python
"""Golden fixtures for the NeuS variant's TRAINING backward, from the REAL reference's autograd.

Run in the build container only (needs /root/reference):

    python tests/golden/make_neus_train_golden.py

The reference's NeuS (neddf/network/neus.py) inside its NeRFRender, grad mode, recorded uniforms (RandFeeder), and the
objective of config/loss/nerf_loss.yaml - the reference's own ColorLoss (weight 1.0, coarse 0.1) and MaskBCELoss (0.05,
0.005), summed as nerf_trainer.py:118-121 - on recorded random targets.  The networks' parameters are not stored: they
are set from seeds by tests/neus_train_oracle.py::seeded_state_dict (a platform-independent integer hash), and the
fixture keeps the seeds (`weight_seed_<tag>`).  Stored in case_neus_train_<name>.npz: configuration, seeds, inputs,
targets, the loss, the integrated outputs, the reference's rays and coarse / fine edge distances, the field outputs
and the upstream gradients that reach them in each pass (d loss / d density [B,S], d loss / d color [B,S,3], captured
with tensor hooks; the renderer does not read `sdf`, so no gradient reaches it) and the parameter gradients,
`variance` included (of the big matrices every 16th output row and 4th input column, neus_train_oracle.fixture_sample).
  relu     config/network/neus.yaml (ReLU, ranks 6 / 4, 8 + 8 layers, skip 4) under config/render/nerf_render.yaml
           (64 + 128 samples, point sampling, separate coarse network)
  tanhexp  tanhExp, ranks 5 / 3, 6 SDF layers with skips [1, 3], 4 colour layers, one network for both passes, cone
           sampling, other sample counts
The tanhexp file also carries `probe_x` / `probe_d2`: the second derivative that double backward finds through the
reference's tanhExp Function (nn_module/tanh_exp.py) at a few x - ex (1 - tx^2), not the true one, because the
Function saves ex and tx without a graph.
"""
import importlib.util
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (sets sys.path for the reference + stubs)

import numpy as np  # noqa: E402
import torch  # noqa: E402
# tests/neus_train_oracle.py by path: on this sys.path `tests` is the reference's own test package
_spec = importlib.util.spec_from_file_location("neus_train_oracle", os.path.join(os.path.dirname(HERE), "neus_train_oracle.py"))
nto = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(nto)
fixture_sample, seeded_state_dict = nto.fixture_sample, nto.seeded_state_dict
from neddf.loss import ColorLoss, MaskBCELoss  # noqa: E402  (reference)
from neddf.nn_module.tanh_exp import tanhExp  # noqa: E402  (reference)

CASES = {
    "relu": dict(
        net={"_target_": "neddf.network.NeuS", "embed_pos_rank": 6, "embed_dir_rank": 4, "sdf_layer_count": 8,
             "sdf_layer_width": 256, "col_layer_count": 8, "col_layer_width": 256, "init_variance": 0.3,
             "activation_type": "ReLU", "skips": [4]},
        render={"sample_coarse": 64, "sample_fine": 128, "dist_near": 2.0, "dist_far": 6.0, "max_dist": 6.0,
                "use_coarse_network": True, "sampling_type": "point"},
        seed=41, rays=2),
    "tanhexp": dict(
        net={"_target_": "neddf.network.NeuS", "embed_pos_rank": 5, "embed_dir_rank": 3, "sdf_layer_count": 6,
             "sdf_layer_width": 256, "col_layer_count": 4, "col_layer_width": 256, "init_variance": 0.45,
             "activation_type": "tanhExp", "skips": [1, 3]},
        render={"sample_coarse": 24, "sample_fine": 40, "dist_near": 1.5, "dist_far": 5.0, "max_dist": 5.5,
                "use_coarse_network": False, "sampling_type": "cone"},
        seed=42, rays=3),
}
PROBE_X = [-3.0, -1.0, -0.25, 0.0, 0.5, 2.0, 21.0]


def tanhexp_probe():
    x = torch.tensor(PROBE_X, dtype=torch.float32, requires_grad=True)
    (d1,) = torch.autograd.grad(tanhExp.apply(x).sum(), x, create_graph=True)
    (d2,) = torch.autograd.grad(d1.sum(), x)
    return np.array(PROBE_X, np.float32), d2.detach().numpy()


def main():
    for name, c in CASES.items():
        torch.manual_seed(c["seed"])
        render = mg.build_render(c["net"], c["render"])
        nc = mg.orc.NeusConfig.from_dict(c["net"])
        seeds = {"fine": c["seed"]}
        if render.network_coarse is not render.network_fine:
            seeds["coarse"] = c["seed"] + 1
        for tag, seed in seeds.items():
            sd = {k: torch.from_numpy(v) for k, v in seeded_state_dict(nc, seed).items()}
            getattr(render, "network_" + tag).load_state_dict(sd)
        cam = mg.synthetic_camera(c["seed"])
        g = torch.Generator().manual_seed(c["seed"])
        B = c["rays"]
        uv = torch.stack([torch.randint(300, 500, (B,), generator=g), torch.randint(300, 500, (B,), generator=g)], 1)
        u_c = torch.rand(B, render.sample_coarse + 1, generator=g)
        u_f = torch.rand(B, render.sample_fine + 1, generator=g)
        targets = {"color": torch.rand(B, 3, generator=g), "mask": (torch.rand(B, generator=g) > 0.5).float()}
        render.set_iter(-1)
        fields, ups, hooks, seen = [], [], [], set()

        def fwd_hook(m, i, o):
            fields.append({k: v.detach().clone() for k, v in o.items()})
            slot = {}
            ups.append(slot)
            for k, v in o.items():
                if v.requires_grad:
                    v.register_hook(lambda gr, k=k, slot=slot: slot.__setitem__(k, gr.detach().clone()))

        for net in (render.network_coarse, render.network_fine):
            if id(net) not in seen:
                seen.add(id(net))
                hooks.append(net.register_forward_hook(fwd_hook))
        # the rays and coarse edge distances the reference's network saw, so that the tests evaluate the very same
        # sample positions (recomputed positions can differ from them in the last bit, and with ReLU a sample within
        # rounding of a kink then lands on the other side)
        seen_rays, seen_dists = [], []
        orig_create = cam.create_rays

        def create_rays(*a, **k):
            rays = orig_create(*a, **k)
            seen_rays.append((rays.ray_dir.detach().clone(), rays.ray_orig.detach().clone()))
            for meth in ("get_sampling_points", "get_sampling_cones"):
                f = getattr(rays, meth)
                setattr(rays, meth, lambda dists, *aa, _f=f, **kk: (seen_dists.append(dists.detach().clone()) or _f(dists, *aa, **kk)))
            return rays

        cam.create_rays = create_rays
        pdf_out = []
        orig_pdf = render.sample_pdf
        render.sample_pdf = lambda *a, **k: (pdf_out.append(orig_pdf(*a, **k).detach().clone()) or pdf_out[-1])
        with mg.RandFeeder([u_c, u_f]):
            with torch.set_grad_enabled(True):
                out = render.render_rays(uv, cam)
        render.sample_pdf = orig_pdf
        cam.create_rays = orig_create
        for h in hooks:
            h.remove()
        loss_dict = {}
        for fn in (ColorLoss(weight=1.0, weight_coarse=0.1), MaskBCELoss(weight=0.05, weight_coarse=0.005)):
            loss_dict.update(fn(out, targets))
        loss = torch.sum(torch.stack(list(loss_dict.values())))  # nerf_trainer.py:118-121
        render.zero_grad()
        loss.backward()
        res = dict(uv=uv.numpy(), u_coarse=u_c.numpy(), u_fine=u_f.numpy(), loss=loss.detach().numpy(),
                   target_color=targets["color"].numpy(), target_mask=targets["mask"].numpy(), dists_fine=pdf_out[0].numpy(),
                   ray_dir=seen_rays[0][0].numpy(), ray_orig=seen_rays[0][1].numpy(), dists_coarse=seen_dists[0].numpy(),
                   **mg.cam_arrays(cam))
        for k, v in out.items():
            res["out_" + k] = v.detach().numpy()
        for tag, f, u in zip(("coarse", "fine"), fields, ups):
            for k, v in f.items():
                res[f"field_{tag}_{k}"] = v.numpy()
            for k, v in u.items():
                res[f"up_{tag}_{k}"] = v.numpy()
        for n, p in render.named_parameters():
            gr = p.grad.detach().numpy()
            res["grad_" + n] = fixture_sample(gr)
        res["cfg"] = json.dumps({"net": c["net"], "render": c["render"], "seed": c["seed"]})
        for tag, seed in seeds.items():
            res[f"weight_seed_{tag}"] = np.array(seed, np.int64)
        if name == "tanhexp":
            res["probe_x"], res["probe_d2"] = tanhexp_probe()
        np.savez_compressed(os.path.join(HERE, f"case_neus_train_{name}.npz"), **res)
        print(name, float(loss.detach()), {k: getattr(v, "shape", None) for k, v in res.items() if k.startswith(("up_", "field_"))})


if __name__ == "__main__":
    main()
