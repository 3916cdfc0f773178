"""CPU: the operand-precision model behind the tensor-core engine (DESIGN.md 4.1), emulated on the
oracle: which splits of the GEMM operands keep NeDDF.forward within the 1e-4 parity bar.

fp16 hi/lo with three products (what csrc/field_tc.cu issues) is as good as fp32; dropping a
product is not, and bf16 parts cost 10x - the measurements that ruled the cheaper variants out."""
import math

import pytest
import torch

from oracle import neddf_oracle as orc
from tests.helpers import PARITY_TOL, nerr


def _case(seed=3, n=1024):
    cfg = orc.FieldConfig()
    P = orc.init_params(cfg, seed=seed, bias_std=0.1)
    st = orc.FieldState()
    g = torch.Generator().manual_seed(seed)
    pos = (torch.rand(n, 1, 3, generator=g) * 2 - 1) * 1.2
    dirs = torch.nn.functional.normalize(torch.randn(n, 1, 3, generator=g), dim=-1)
    var = torch.rand(n, 1, 3, generator=g) * 1e-3
    return cfg, P, st, pos, dirs, var


def _errors(mm):
    cfg, P, st, pos, dirs, var = _case()
    ref = orc.field_forward(P, cfg, st, pos, dirs, var)
    out = orc.field_forward(P, cfg, st, pos, dirs, var, mm=mm)
    return {k: nerr(out[k].numpy(), ref[k].numpy()) for k in ("density", "color", "distance")}


def _h(t):
    return t.to(torch.float16).to(torch.float32)


def test_fp16_three_products_is_fp32_grade():
    e = _errors(orc.split_matmul("fp16", 3))
    assert max(e.values()) < 0.1 * PARITY_TOL, e
    t = _errors(orc.split_matmul("tf32", 3))
    assert max(e.values()) < 3 * max(t.values()) + 1e-6, (e, t)  # as accurate as 3xTF32 at twice its tensor rate


@pytest.mark.parametrize("variant", ["single fp16 product", "weights hi only", "activations hi only"])
def test_cheaper_operand_splits_miss_the_bar(variant):
    def mm(a, b):  # a = activations, b = weights
        ah, bh = _h(a), _h(b)
        al, bl = _h(a - ah), _h(b - bh)
        if variant == "single fp16 product":
            return ah @ bh
        if variant == "weights hi only":
            return ah @ bh + al @ bh
        return ah @ bh + ah @ bl
    e = _errors(mm)
    assert max(e.values()) > PARITY_TOL, (variant, e)


def test_bf16_parts_cost_an_order_of_magnitude():
    """bf16 hi/lo (16 mantissa bits in total) stays inside the bar on its own but is ~10x worse than
    fp16 hi/lo (22 bits) at the same tensor rate - no reason to use it."""
    b, h = _errors(orc.split_matmul("bf16", 3)), _errors(orc.split_matmul("fp16", 3))
    assert max(b.values()) > 5 * max(h.values()), (b, h)


def test_fp8_lo_weights_keep_the_bar_but_not_the_margin():
    """lo parts of the weights as e4m3 * 2^S (25 % fewer weight bytes): inside 1e-4 on smooth
    configurations but 5-20x worse than fp16 lo parts; on hardware it was no faster and broke the
    kinked (ReLU / point-sampling) case - rejected."""
    cfg, P, *_ = _case()
    maxlo = max(float((v - _h(v)).abs().max()) for k, v in P.items() if k.endswith("weight"))
    S = min(24, math.floor(math.log2(240 / maxlo)))

    def mm(a, b):
        ah, bh = _h(a), _h(b)
        al = _h(a - ah)
        bl = ((b - bh) * 2.0 ** S).to(torch.float8_e4m3fn).to(torch.float32) * 2.0 ** -S
        return ah @ bh + al @ bh + ah @ _h(bl)
    e8, e16 = _errors(mm), _errors(orc.split_matmul("fp16", 3))
    assert max(e8.values()) < PARITY_TOL and max(e8.values()) > 3 * max(e16.values()), (e8, e16)
