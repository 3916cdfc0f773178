"""Per-phase cycle breakdown of the tensor-core field kernel (engines "tc" and "tc2").

Builds a copy of the library whose field_tc.cu is compiled with -DNEDDF_TC_PHASE_CLOCKS (in a temporary
directory, linked against the in-tree objects of the normal build), renders a slice of the bench frame
(131,072 rays of bench camera 0 by default, coarse and fine launches) and prints the mean cycles per
32-sample tile that consumer thread 0 of each CTA spent in every phase:

  prologue   geometry + scaled position embedding of the tile
  distance   distance-trunk MMAs and epilogues
  heads      distance / aux head with the colour-trunk inputs, and the colour head with the outputs
  colour     colour-trunk MMAs and epilogues
  park       images-only launches: parking a tile's colour-trunk operand and loading a group's back

If NEDDF_B200_LIB is set, that library is used as it is (it must have been built with the define).

usage: python tools/tc_phase_clocks.py [n_rays] [engine ...]
"""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ("prologue", "distance", "heads", "colour", "park")


def build_instrumented(out_dir):
    import __graft_entry__ as ge
    # the other objects of the library, in-tree as the normal build leaves them; built in a child process, since
    # build() imports the package, and this process has to import it only after pointing NEDDF_B200_LIB at the copy
    subprocess.run([sys.executable, os.path.join(ROOT, "__graft_entry__.py")], check=True, stdout=subprocess.DEVNULL)
    csrc = ge.CSRC
    obj = os.path.join(out_dir, "field_tc_clocks.o")
    lib = os.path.join(out_dir, "libneddf_b200_clocks.so")
    subprocess.run([ge._nvcc()] + ge.NVCC_FLAGS + ["-DNEDDF_TC_PHASE_CLOCKS", "-c", os.path.join(csrc, "field_tc.cu"),
                    "-o", obj], check=True)
    objs = [obj if s == "field_tc.cu" else os.path.join(csrc, s.replace(".cu", ".o")) for s in ge.SOURCES]
    subprocess.run([ge._nvcc(), "-shared", "-o", lib] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"],
                   check=True)
    return lib


def main():
    n_rays = int(sys.argv[1]) if len(sys.argv) > 1 else 131072
    engines = sys.argv[2:] or ["tc", "tc2"]
    tmp = tempfile.TemporaryDirectory(prefix="neddf_phase_")
    if not os.environ.get("NEDDF_B200_LIB"):
        os.environ["NEDDF_B200_LIB"] = build_instrumented(tmp.name)
    import torch
    import bench
    import neddf_b200
    from neddf_b200 import _lib

    assert _lib.LIB_PATH == os.environ["NEDDF_B200_LIB"], "the package was imported before the library was chosen"
    read = _lib.lib().neddf_tc_phase_clocks
    read.restype, read.argtypes = C.c_int32, [C.POINTER(C.c_ulonglong)]
    sums = (C.c_ulonglong * (len(PHASES) + 1))()

    dev = torch.device("cuda:0")
    sd, _ = bench.seeded_state_dict()
    R, T, calib = bench.synthetic_pose(0)
    cam = neddf_b200.Camera.from_matrix(neddf_b200.PinholeCalib(calib), R, T).to(dev)
    cam.update_transform()
    first = (bench.H // 2) * bench.W
    for engine in engines:
        render = neddf_b200.NeRFRender(network_config=bench.NET_CFG, **bench.RENDER_CFG)
        render.load_state_dict(sd)
        render.to(dev)
        render.set_iter(-1)
        render.set_engine(engine)
        render.render_pixels(bench.W, bench.H, cam, ["color", "depth"], 1, first, n_rays)  # warm-up
        _lib.check(read(sums), "phase clocks")
        render.render_pixels(bench.W, bench.H, cam, ["color", "depth"], 1, first, n_rays)
        _lib.check(read(sums), "phase clocks")
        tiles = sums[len(PHASES)]
        per_tile = {k: sums[i] / max(tiles, 1) for i, k in enumerate(PHASES)}
        per_tile["total"] = sum(per_tile.values())
        print(f"{engine}: {tiles} tiles, mean cycles per tile (consumer thread 0)")
        for k, v in per_tile.items():
            print(f"  {k:9s} {v:10.0f}  {100 * v / per_tile['total']:5.1f} %")
        print(json.dumps({"engine": engine, "n_rays": n_rays, "tiles": tiles, "gpu": torch.cuda.get_device_name(0),
                          "cycles_per_tile": {k: round(v) for k, v in per_tile.items()}}), flush=True)


if __name__ == "__main__":
    main()
