"""NeRF and NeuS network structures the CUDA-core kernels and their training backward are tested at (CPU and GPU suites).

The goldens of both variants share a few structures; the table below walks what depends on the configuration instead:
the segment tables of ``build_program``, the shared-memory map at the row maxima (NeRF ``kMaxE`` = 64 / ``kMaxD`` = 32,
NeuS ``kMaxE`` = 64 / ``kMaxX`` = 32), skip concatenation at layer 0, consecutive skips and the last skip allowed, the
single-SDF-layer NeuS path, the deepest layer loops (NeRF forward 13, training 12; NeuS 12 + 12), ``n_skips`` at its
bound of 8 and the weight-gradient GEMMs at the operand widths these structures produce.  Each entry holds the
``neddf_b200.NeRF`` / ``neddf_b200.NeuS`` keyword arguments, the ``set_iter`` value of the run, whether the training
handle accepts the structure, and why it is in the table.
"""
import torch

from oracle import neddf_oracle as orc
from tests.field_configs import rays, samples, upstream  # noqa: F401  (the generators of the NeDDF table)

CONFIGS = {
    # --- NeRF (nerf::unsupported: layer_count 2..13, training 2..12; 6 pos <= 64, 6 dir <= 32; <= 8 skips) ---
    "N1_min": dict(
        variant="nerf", kw=dict(embed_pos_rank=1, embed_dir_rank=1, layer_count=2, skips=[],
                                activation_type="LeakyReLU", density_activation_type="tanhExp"),
        iter=-1, train=True, why="fewest layers, smallest embeddings, LeakyReLU hidden with a tanhExp density"),
    "N2_max_embed": dict(
        variant="nerf", kw=dict(embed_pos_rank=10, embed_dir_rank=5, layer_count=4, skips=[0],
                                activation_type="tanhExp", density_activation_type="ReLU"),
        iter=-1, train=True, why="60 + 30 embedding rows (kMaxE, kMaxD edges); skip right after layer 0 (316 = 256 + 60)"),
    "N3_deep_fwd": dict(
        variant="nerf", kw=dict(embed_pos_rank=6, embed_dir_rank=2, layer_count=13, skips=[0, 5, 11],
                                activation_type="ReLU", density_activation_type="LeakyReLU"),
        iter=-1, train=False, why="the forward's 13 layers, which the training handle refuses; 11 is the last skip allowed"),
    "N4_deep_train": dict(
        variant="nerf", kw=dict(embed_pos_rank=10, embed_dir_rank=4, layer_count=12, skips=[1, 2, 10],
                                activation_type="tanhExp", density_activation_type="tanhExp"),
        iter=-1, train=True, why="the training backward's 12 layers; consecutive skips"),
    "N5_eight_skips": dict(
        variant="nerf", kw=dict(embed_pos_rank=4, embed_dir_rank=2, layer_count=10, skips=[0, 1, 2, 3, 4, 5, 6, 7],
                                activation_type="LeakyReLU", density_activation_type="LeakyReLU"),
        iter=-1, train=True, why="n_skips at its bound: layers 1..8 all take two segments"),
    "N6_warmup": dict(
        variant="nerf", kw=dict(lowpass_alpha_offset=2.0),
        iter=1500, train=True, why="default structure in the low-pass window: alpha 3.5 weights frequency 3 by half"),
    # --- NeuS (neus::unsupported: sdf / col 1..12; 6 pos <= 64, 6 + 6 dir <= 32; <= 8 skips, none on the last SDF layer) ---
    "S1_one_sdf": dict(
        variant="neus", kw=dict(embed_pos_rank=1, embed_dir_rank=1, sdf_layer_count=1, col_layer_count=1, skips=[],
                                activation_type="ReLU"),
        iter=-1, train=True, why="sdf is channel 0 of the first layer; shortest colour trunk"),
    "S2_max_embed": dict(
        variant="neus", kw=dict(embed_pos_rank=10, embed_dir_rank=4, sdf_layer_count=2, col_layer_count=1, skips=[0],
                                activation_type="tanhExp"),
        iter=-1, train=True, why="60 embedding rows; colour input head at 30 of kMaxX = 32 (286 = 256 + 30 columns)"),
    "S3_deepest": dict(
        variant="neus", kw=dict(embed_pos_rank=6, embed_dir_rank=2, sdf_layer_count=12, col_layer_count=12, skips=[0, 5, 10],
                                activation_type="tanhExp"),
        iter=-1, train=True, why="both trunks at kMaxSdf / kMaxCol; 10 is the last skip allowed"),
    "S4_eight_skips": dict(
        variant="neus", kw=dict(embed_pos_rank=4, embed_dir_rank=3, sdf_layer_count=10, col_layer_count=2,
                                skips=[0, 1, 2, 3, 4, 5, 6, 7], activation_type="ReLU"),
        iter=-1, train=True, why="n_skips at its bound; ReLU normals through every layer"),
    "S5_sharp": dict(
        variant="neus", kw=dict(embed_pos_rank=10, embed_dir_rank=4, sdf_layer_count=2, col_layer_count=1, skips=[0],
                                activation_type="tanhExp", init_variance=2.0),
        iter=-1, train=True, sharpen=True,
        why="sdf from its floor (tanhExp ~ -0.35) to above 5: exp(-20 sdf) underflows to 0 at one end, a steep peak at 0"),
}

NAMES = list(CONFIGS)
NERF = [n for n in NAMES if CONFIGS[n]["variant"] == "nerf"]
NEUS = [n for n in NAMES if CONFIGS[n]["variant"] == "neus"]
TRAIN = [n for n in NAMES if CONFIGS[n]["train"]]
SEED = {name: 7300 + i for i, name in enumerate(NAMES)}
# S5: the 5 % and 75 % quantiles of the sdf channel's pre-activation over `samples` positions go to -1.2 (tanhExp's
# minimum, -0.353, sits at -1.1) and 5.5 (past 5.2, exp(-20 sdf) is below fp32's smallest subnormal)
SHARP_SDF = ((0.05, -1.2), (0.75, 5.5))


def variant(name) -> str:
    return CONFIGS[name]["variant"]


def kwargs(name):
    """Constructor keyword arguments (fresh copies: the module keeps what it is given)."""
    kw = dict(CONFIGS[name]["kw"])
    if "skips" in kw:
        kw["skips"] = list(kw["skips"])
    return kw


def config(name):
    """orc.NerfConfig / orc.NeusConfig of the entry."""
    return (orc.NerfConfig if variant(name) == "nerf" else orc.NeusConfig)(**kwargs(name))


def layer_shapes(name):
    return (orc.nerf_layer_shapes if variant(name) == "nerf" else orc.neus_layer_shapes)(config(name))


def lowpass_alpha(name) -> float:
    """NeRF.set_iter's low-pass alpha at the entry's iteration."""
    return config(name).lowpass_alpha_at(CONFIGS[name]["iter"])


def kinked(name) -> bool:
    return CONFIGS[name]["kw"].get("activation_type", "ReLU") in ("ReLU", "LeakyReLU")


def params(name):
    """Seeded oracle parameters ([in,out] weights) with perturbed biases, so that the bias path is live.  S5 widens and
    lifts the sdf channel (``layers_sdf.1``, column 0) as SHARP_SDF says."""
    cfg = config(name)
    if variant(name) == "nerf":
        return orc.nerf_init_params(cfg, SEED[name], bias_std=0.05)
    P = orc.neus_init_params(cfg, SEED[name], bias_std=0.05)
    if CONFIGS[name].get("sharpen"):
        last = f"layers_sdf.{cfg.sdf_layer_count - 1}"
        pos, _, _ = samples(1, 4096, SEED[name])
        hx = orc.pe_plain(pos.reshape(-1, 3).double(), cfg.embed_pos_rank)
        for lid in range(cfg.sdf_layer_count - 1):
            hx = orc.density_act("tanhExp", hx @ P[f"layers_sdf.{lid}.weight"].double() + P[f"layers_sdf.{lid}.bias"].double())
            if lid in cfg.skips:
                hx = torch.cat([hx, orc.pe_plain(pos.reshape(-1, 3).double(), cfg.embed_pos_rank)], 1)
        z = hx @ P[f"{last}.weight"][:, 0].double()
        (q0, v0), (q1, v1) = SHARP_SDF
        z0, z1 = (float(torch.quantile(z, q)) for q in (q0, q1))
        a = (v1 - v0) / (z1 - z0)
        P[f"{last}.weight"][:, 0] *= a
        P[f"{last}.bias"][0] = v0 - a * z0
    return P


def state_dict(name):
    """``params`` in the modules' layout: torch Linear weights [out,in]."""
    return {k: (v.t().contiguous() if k.endswith(".weight") else v.clone()) for k, v in params(name).items()}

