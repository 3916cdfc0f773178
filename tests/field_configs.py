"""NeDDF network structures the field engines and the training backward are tested at (CPU and GPU suites).

Every golden case shares one structure (ranks 10/4, 8 + 4 layers, skip 4); the table below walks the tables that
depend on the configuration instead: the layer / segment table of ``neddf_field_create``, the tensor-core AUX layout
(``n_e0 = 6 pos <= 64``, ``off_h = 6 (pos + dir) + 3 <= 96``), skip handling, the low-pass window and the 128-column
tiling of the weight-gradient GEMMs.  Each entry holds ``orc.FieldConfig`` / ``neddf_b200.NeDDF`` keyword arguments,
the ``set_iter`` value of the run and the engines that cover it.
"""
import torch

from oracle import neddf_oracle as orc

TC_ENGINES = ("fp32", "tc", "tc2")
FP32_ONLY = ("fp32",)

CONFIGS = {
    # NeDDF() as constructed: 7 + 7 = 14 hidden layers
    "C1_default": dict(
        kw=dict(embed_pos_rank=10, embed_dir_rank=4, ddf_layer_count=8, col_layer_count=8, skips=[4],
                activation_type="tanhExp", density_activation_type="ReLU"),
        iter=-1, engines=TC_ENGINES),
    # no hidden-to-hidden layer in either trunk; n_e0 = 6, off_h = 15
    "C2_minimal": dict(
        kw=dict(embed_pos_rank=1, embed_dir_rank=1, ddf_layer_count=2, col_layer_count=2, skips=[],
                activation_type="LeakyReLU", density_activation_type="tanhExp"),
        iter=-1, engines=TC_ENGINES),
    # off_h = 93, the largest colour input the tensor-core AUX takes; skip at layer 0
    "C3_aux_edge": dict(
        kw=dict(embed_pos_rank=10, embed_dir_rank=5, ddf_layer_count=4, col_layer_count=2, skips=[0],
                activation_type="ReLU", density_activation_type="LeakyReLU"),
        iter=-1, engines=TC_ENGINES),
    # n_e0 = 66 > 64: the tensor-core engines refuse, "auto" runs fp32; consecutive skips
    "C4_past_es": dict(
        kw=dict(embed_pos_rank=11, embed_dir_rank=1, ddf_layer_count=5, col_layer_count=3, skips=[1, 2],
                activation_type="tanhExp", density_activation_type="LeakyReLU"),
        iter=-1, engines=FP32_ONLY),
    # off_h = 99 > 96 with n_e0 = 48: refused by the AUX bound alone
    "C5_past_aux": dict(
        kw=dict(embed_pos_rank=8, embed_dir_rank=8, ddf_layer_count=3, col_layer_count=3, skips=[0],
                activation_type="ReLU", density_activation_type="ReLU"),
        iter=-1, engines=FP32_ONLY),
    # ranks at the fp32 engine's limit: k_total = 547 (~204 KB of shared memory); colour input 195 = 128 + 67 columns
    # in the weight-gradient GEMM; skip at ddf_layer_count - 3, the last one allowed
    "C6_fp32_limit": dict(
        kw=dict(embed_pos_rank=16, embed_dir_rank=16, ddf_layer_count=6, col_layer_count=2, skips=[0, 3],
                activation_type="tanhExp", density_activation_type="tanhExp"),
        iter=-1, engines=FP32_ONLY),
    # 12 + 12 = 24 hidden layers, the most a field describes (kMaxHidden); three skips
    "C7_deepest": dict(
        kw=dict(embed_pos_rank=6, embed_dir_rank=2, ddf_layer_count=13, col_layer_count=13, skips=[0, 5, 10],
                activation_type="LeakyReLU", density_activation_type="LeakyReLU"),
        iter=-1, engines=TC_ENGINES),
    # warm-up state: lowpass_alpha = 2 + 1.5 = 3.5 (half weight on frequency 3, 1e-7 above), aux_grad_scale = 0.15;
    # a zero penalty weight and a missing key (weighted 1.0)
    "C8_warmup": dict(
        kw=dict(embed_pos_rank=10, embed_dir_rank=4, ddf_layer_count=8, col_layer_count=4, skips=[4],
                activation_type="LeakyReLU", density_activation_type="ReLU", lowpass_alpha_offset=2.0,
                penalty_weight={"constraints_aux_grad": 0.05, "constraints_dDdt": 0.0, "constraints_color": 0.01,
                                "range_distance": 1.0}),
        iter=1500, engines=TC_ENGINES),
}

NAMES = list(CONFIGS)
PAIRS = [(name, engine) for name in NAMES for engine in CONFIGS[name]["engines"]]
SEED = {name: 7100 + i for i, name in enumerate(NAMES)}


def kwargs(name):
    """Constructor keyword arguments (fresh copies: the module keeps what it is given)."""
    kw = dict(CONFIGS[name]["kw"])
    kw["skips"] = list(kw["skips"])
    if "penalty_weight" in kw:
        kw["penalty_weight"] = dict(kw["penalty_weight"])
    return kw


def field_config(name) -> orc.FieldConfig:
    return orc.FieldConfig(**kwargs(name))


def state(name) -> orc.FieldState:
    return orc.FieldState.at_iter(field_config(name), CONFIGS[name]["iter"])


def params(name):
    """Seeded parameters with perturbed biases (so the bias path is live)."""
    return orc.init_params(field_config(name), SEED[name], bias_std=0.05)


def kinked(name) -> bool:
    return CONFIGS[name]["kw"]["activation_type"] in ("ReLU", "LeakyReLU")


def samples(B, S, seed):
    """Sampling tensors [B,S,3] (fp32): positions in the unit cube's neighbourhood, unit directions and small
    cone variances."""
    g = torch.Generator().manual_seed(seed)
    pos = (torch.rand(B, S, 3, generator=g) - 0.5) * 2.2
    dirs = torch.nn.functional.normalize(torch.randn(B, S, 3, generator=g), dim=-1)
    var = torch.rand(B, S, 3, generator=g) * 1e-3
    return pos, dirs, var


def rays(B, S, seed):
    """(ray_dir [B,3], ray_orig [B,3], dists [B,S]) (fp32): rays from a sphere of radius 3 through the unit cube,
    sorted edge distances in [1.5, 4.5]."""
    g = torch.Generator().manual_seed(seed)
    orig = 3.0 * torch.nn.functional.normalize(torch.randn(B, 3, generator=g), dim=-1)
    target = (torch.rand(B, 3, generator=g) - 0.5) * 0.8
    ray_dir = torch.nn.functional.normalize(target - orig, dim=-1)
    dists = torch.sort(1.5 + 3.0 * torch.rand(B, S, generator=g), dim=1).values
    return ray_dir.contiguous(), orig.contiguous(), dists.contiguous()


def upstream(B, S, seed):
    """Random upstream gradients of density [B,S], colour [B,S,3] and fields_penalty [B,S] (fp32)."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, S, generator=g), torch.randn(B, S, 3, generator=g), torch.randn(B, S, generator=g)
