"""NeRF variant, training backward on the GPU: csrc/nerf_train.cu against the real reference's autograd gradients (see
tests/nerf_train_gpu_child.py for the checks).  Each check runs in a CHILD PROCESS with a timeout and this file is
collected last, so that a fault or a hang of the opt-in kernel cannot poison the CUDA context of the rest of the suite;
a failing check fails the suite.  tests/test_nerf_neus_configs_gpu.py holds the same backward at other structures."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("case", ["relu", "tanhexp"])
@pytest.mark.parametrize("check", ["field", "render"])
def test_nerf_training_backward_on_hardware(check, case):
    r = subprocess.run([sys.executable, "-m", "tests.nerf_train_gpu_child", check, case], cwd=ROOT, capture_output=True, text=True,
                       timeout=240)
    print(r.stdout[-2000:], r.stderr[-3000:])
    assert r.returncode == 0 and f"{check} {case} ok" in r.stdout
