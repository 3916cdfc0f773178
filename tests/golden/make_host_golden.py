"""Golden data of three host-side comparisons with the REAL reference, so that the tests that use it need no
reference checkout:

* case_neus_init.npz: neddf.network.NeuS(**NEUS_KW) built right after torch.manual_seed(7): the state_dict keys in
  order, every tensor's shape and float64 sum, and the values at 64 seeded positions of every tensor;
* case_trainer_gather.npz: BaseTrainer.construct_ground_truth (neddf/trainer/base_trainer.py:205-245) on a seeded
  dataset entry and seeded pixel ids;
* case_bunny_checkpoint.npz: the saved hydra config of pretrained/bunny_smoke (its render / network nodes, JSON) and
  the state_dict of models/model_02000.pth as keys in order, shapes and float64 sums.

    python tests/golden/make_host_golden.py <reference checkout>   ->  tests/golden/case_neus_init.npz,
                                                                      tests/golden/case_trainer_gather.npz,
                                                                      tests/golden/case_bunny_checkpoint.npz
"""
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
NEUS_KW = dict(embed_pos_rank=5, embed_dir_rank=3, sdf_layer_count=6, col_layer_count=3, activation_type="tanhExp",
               init_variance=0.45, skips=[1, 3])
N_SAMPLE = 64
GATHER_KINDS = ["ColorLoss", "MaskBCELoss", "FieldsConstraintLoss"]


def neus_fingerprint(sd):
    """(keys, shapes, float64 sums, sampled values) of a state_dict; the sample positions depend on the shape only."""
    keys = list(sd)
    shapes, sums, samples = [], [], []
    for k in keys:
        t = sd[k].detach().to(torch.float64).reshape(-1)
        shapes.append(list(sd[k].shape) + [-1] * (2 - sd[k].dim()))
        sums.append(float(t.sum()))
        idx = np.random.default_rng(t.numel()).integers(0, t.numel(), N_SAMPLE)
        samples.append(t.numpy()[idx])
    return keys, np.array(shapes, np.int64), np.array(sums), np.stack(samples)


def gather_inputs():
    rng = np.random.default_rng(3)
    rgb = rng.integers(0, 256, (20, 30, 3), dtype=np.uint8)
    mask = rng.integers(0, 256, (20, 30), dtype=np.uint8)
    g = torch.Generator().manual_seed(5)
    us = (torch.rand(64, generator=g) * 29).to(torch.int16)
    vs = (torch.rand(64, generator=g) * 19).to(torch.int16)
    return rgb, mask, us, vs


def main(ref):
    sys.path.insert(0, os.path.join(HERE, "_refstub"))
    sys.path.insert(0, ref)
    # the trainer module imports skimage.metrics at module level; nothing of it is used here
    sk, m = types.ModuleType("skimage"), types.ModuleType("skimage.metrics")
    m.peak_signal_noise_ratio = m.structural_similarity = None
    sk.metrics = m
    sys.modules["skimage"], sys.modules["skimage.metrics"] = sk, m
    from neddf.network import NeuS
    from neddf.trainer.base_trainer import BaseTrainer

    torch.manual_seed(7)
    keys, shapes, sums, samples = neus_fingerprint(NeuS(**NEUS_KW).state_dict())
    np.savez(os.path.join(HERE, "case_neus_init.npz"), keys=np.array(keys), shapes=shapes, sums=sums, samples=samples)

    rgb, mask, us, vs = gather_inputs()

    class T:
        pass

    t = T()
    t.device = torch.device("cpu")
    t.dataset = [dict(rgb_images=rgb, mask_images=mask)]
    out = BaseTrainer.construct_ground_truth(t, 0, us, vs, GATHER_KINDS)
    np.savez(os.path.join(HERE, "case_trainer_gather.npz"), rgb=rgb, mask=mask, us=us.numpy(), vs=vs.numpy(),
             keys=np.array(sorted(out)), **{"out_" + k: v.numpy() for k, v in out.items()},
             **{"dtype_" + k: np.array(str(v.dtype)) for k, v in out.items()})
    import yaml
    run = os.path.join(ref, "pretrained", "bunny_smoke")
    cfg = yaml.safe_load(open(os.path.join(run, ".hydra", "config.yaml")))
    ckpt = torch.load(os.path.join(run, "models", "model_02000.pth"), map_location="cpu")
    keys, shapes, sums, _ = neus_fingerprint(ckpt)
    np.savez(os.path.join(HERE, "case_bunny_checkpoint.npz"), render=np.array(json.dumps(cfg["render"])),
             network=np.array(json.dumps(cfg["network"])), keys=np.array(keys), shapes=shapes, sums=sums)
    print("wrote case_neus_init.npz, case_trainer_gather.npz, case_bunny_checkpoint.npz")


if __name__ == "__main__":
    main(sys.argv[1])
