#!/usr/bin/env python
"""Golden fixture for the device grid behind BaseNeuralField.voxelize / extract_mesh, from the REAL reference.

Needs a checkout of the reference where make_golden.py looks for it:

    python tests/golden/make_mesh_golden.py

Builds the reference's NeRFRender with the bunny_smoke config and checkpoint weights (bunny_smoke_weights.npz, the
config stored in case_bunny.npz) and calls its ``get_network().voxelize("distance", cube_range=1.1,
cube_resolution=32)`` the way scripts/fields_visualizer.py:528-541 does: constructor state, no set_iter.  The
32^3 fp32 volume goes to case_mesh_bunny.npz.  It pins the grid's point order and axis order against the reference
itself.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (sets sys.path for the reference + stubs)

import numpy as np  # noqa: E402
import torch  # noqa: E402

CUBE_RANGE = 1.1
RESOLUTION = 32


def main():
    meta = json.loads(str(np.load(os.path.join(HERE, "case_bunny.npz"))["cfg"]))
    render = mg.build_render(meta["network"], meta["render"])
    wz = np.load(os.path.join(HERE, meta["weights"]))
    sd = {}
    for tag in ("fine", "coarse"):
        sd.update({f"network_{tag}.{k}": torch.from_numpy(wz[k]) for k in wz.files})
    print("bunny load:", render.load_state_dict(sd))
    vol = render.get_network().voxelize(field_name="distance", cube_range=CUBE_RANGE, cube_resolution=RESOLUTION)
    assert vol.dtype == np.float32 and vol.shape == (RESOLUTION,) * 3
    np.savez_compressed(os.path.join(HERE, "case_mesh_bunny.npz"), volume=vol, field=np.array("distance"),
                        cube_range=np.float64(CUBE_RANGE), cube_resolution=np.int64(RESOLUTION))
    print("case_mesh_bunny:", float(vol.min()), float(vol.max()), "inside 0.0275:", int((vol < 0.0275).sum()))


if __name__ == "__main__":
    main()
