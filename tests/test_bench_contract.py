"""bench.py contract checks that run without a GPU: the reference arm's JSON line (oracle port on
host cores) and the workload constants BASELINE.json quotes."""
import json
import os
import subprocess
import sys

import pytest


def test_reference_arm_prints_one_json_line(repo_root):
    env = dict(os.environ, OMP_NUM_THREADS="4")
    out = subprocess.run([sys.executable, os.path.join(repo_root, "bench.py"), "--impl", "reference", "--steps", "1",
                          "--warmup", "3", "--cpu-rays", "4"], capture_output=True, text=True, timeout=600, env=env,
                         cwd=repo_root)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    j = json.loads(lines[0])
    assert j["impl"] == "reference" and j["unit"] == "ray-samples/s" and j["higher_is_better"] is True
    assert j["metric"] == "ray-samples/s (800x800x192)" and j["value"] > 0 and j["n_gpus"] == 1
    assert j["cpu_baseline"]["kind"] == "port" and j["cpu_baseline"]["value"] == j["value"]
    assert j["e2e"] == {"value": j["value"], "unit": "ray-samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert j["config"]["workload"] and "model" not in j["config"]
    assert j["gpu_launches"] == 0


def test_reference_arm_non_zero_ranks_do_nothing(repo_root):
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    out = subprocess.run([sys.executable, os.path.join(repo_root, "bench.py"), "--impl", "reference", "--gpus", "2"],
                         capture_output=True, text=True, timeout=300, env=env, cwd=repo_root)
    assert out.returncode == 0 and out.stdout.strip() == ""


def test_workload_constants_match_baseline(repo_root):
    sys.path.insert(0, repo_root)
    import bench
    base = json.load(open(os.path.join(repo_root, "BASELINE.json")))
    assert bench.W == 800 and bench.H == 800 and bench.NOMINAL_PER_RAY == 192
    assert bench.EVALS_PER_RAY == 65 + 194  # coarse edges + merged fine edges (nerf_render.py:118-156)
    assert "ray-samples/s" in json.dumps(base)


def test_product_weights_equal_the_oracle_stream(repo_root):
    """bench.py builds its weights without test infrastructure; the CPU legs (oracle) must see the same
    numbers: the product-side generator stream equals oracle.init_params."""
    sys.path.insert(0, repo_root)
    import torch

    import bench
    from oracle import neddf_oracle as orc
    p = bench.seeded_params()
    ref = orc.init_params(orc.FieldConfig.from_dict(bench.NET_CFG), bench.WEIGHT_SEED, bias_std=0.05)
    assert list(p) == list(ref)
    assert all(torch.equal(p[k], ref[k]) for k in ref)
    src = open(os.path.join(repo_root, "bench.py")).read()
    main_src = src[src.index("def main():"):]
    assert "oracle" not in main_src.split("cpu_port_rate")[0]  # product arm set-up imports no oracle

