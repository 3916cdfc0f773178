"""Make the reference's own scripts pick up the CUDA renderer without editing them.

``neddf/scripts/run_eval.py`` re-composes the *saved* hydra config, whose ``_target_`` strings are
always ``neddf.render.NeRFRender`` / ``neddf.network.NeDDF`` (SURVEY 8(b)).  Hydra resolves
those dotted paths by attribute lookup at instantiate time, so rebinding the two attributes on
the already-imported reference package is enough:

    import neddf_b200.install; neddf_b200.install.install()

or, without touching any file of the reference:

    python -m neddf_b200.launch neddf/scripts/run_eval.py pretrained/bunny_smoke
"""
import importlib


def install(patch_trainer: bool = False) -> None:
    """Rebind the reference's render / network classes; with ``patch_trainer`` also replace
    ``BaseTrainer.construct_ground_truth`` by the vectorised gather of ``neddf_b200.trainer_glue`` and the three
    loss classes of ``neddf.loss`` by the fused-kernel ones of ``neddf_b200.losses``."""
    import neddf_b200

    ref_render = importlib.import_module("neddf.render")
    ref_network = importlib.import_module("neddf.network")
    ref_render.NeRFRender = neddf_b200.NeRFRender
    ref_network.NeDDF = neddf_b200.NeDDF
    for mod, name, obj in (("neddf.render.nerf_render", "NeRFRender", neddf_b200.NeRFRender),
                           ("neddf.network.neddf", "NeDDF", neddf_b200.NeDDF)):
        try:
            setattr(importlib.import_module(mod), name, obj)
        except Exception:
            pass
    if patch_trainer:
        from neddf_b200 import eval_io, losses, trainer_glue

        base_trainer = importlib.import_module("neddf.trainer.base_trainer")
        base_trainer.BaseTrainer.construct_ground_truth = trainer_glue.construct_ground_truth
        base_trainer.BaseTrainer.render_all = eval_io.render_all  # uint8 / PNG / PSNR overlapped with the next frame
        # the loss classes hydra instantiates from config/loss/*.yaml (`_target_: neddf.loss.ColorLoss` ...):
        # same constructors and call signature, one CUDA launch each instead of ~10 element-wise kernels
        ref_loss = importlib.import_module("neddf.loss")
        for name in ("ColorLoss", "MaskBCELoss", "FieldsConstraintLoss"):
            setattr(ref_loss, name, getattr(losses, name))
