"""python -m neddf_b200.launch <reference script.py> [args...]: run a reference entry point
(neddf/scripts/run.py, run_eval.py) with NeRFRender / NeDDF rebound to the CUDA classes.
NEDDF_B200_PATCH_TRAINER=1 also swaps in the vectorised ground-truth gather (trainer_glue.py)."""
import os
import runpy
import sys


def main() -> None:
    if len(sys.argv) < 2:
        raise SystemExit(__doc__)
    from .install import install

    install(patch_trainer=os.environ.get("NEDDF_B200_PATCH_TRAINER", "0") not in ("", "0"))
    script = sys.argv[1]
    sys.argv = sys.argv[1:]
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main()
