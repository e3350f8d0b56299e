"""CPU test: the fp32 tensor-core error budgets (tests/tc_budget.py) separate a correct kernel from a kernel that drops one
bf16x3 term.  The emulated kernel must sit at least 3x below the budget on every tensor, and every single-term mutation must
land at least 3x above it on some tensor.  The GPU tests compare the kernels with the fp64 oracle at these budgets."""
import pytest
import torch

import tc_budget as tb

MARGIN = 3.0


def _inputs(B, Cq, C, H, W, scale, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Cq, H, W, generator=g) * scale
    k = torch.randn(B, Cq, H, W, generator=g) * scale
    v = torch.randn(B, C, H, W, generator=g)
    dout = torch.randn(B, C, H, W, generator=g)
    return q, k, v, dout


CASES = [
    # (shape B,Cq,C,H,W, q/k scale, budget, tensors allowed a smaller margin below the budget: {name: margin})
    ((2, 32, 256, 20, 97), 0.7, tb.FP32_BUDGET, {}),
    ((1, 16, 64, 1, 300), 0.7, tb.FP32_BUDGET, {}),
    ((1, 64, 128, 33, 29), 1.0, tb.FP32_BUDGET, {}),
    ((1, 64, 128, 41, 37), 1.5, tb.FP32_PEAKED_BUDGET, {"lse": 2.0}),
]


@pytest.mark.parametrize("shape,scale,budget,relaxed", CASES, ids=[f"{'x'.join(map(str, c[0]))}-s{c[1]}" for c in CASES])
def test_budget_separates_the_kernel_from_single_term_mutations(shape, scale, budget, relaxed):
    q, k, v, dout = _inputs(*shape, scale=scale, seed=sum(shape))
    ref = tb.reference(q, k, v, dout)
    floor = {n: tb.error(n, x, ref[n]) for n, x in tb.emulate(q, k, v, dout).items()}
    for n, e in floor.items():
        assert e * relaxed.get(n, MARGIN) <= budget[n], ("emulated kernel too close to the budget", n, e, budget[n])
    for m in tb.MUTATIONS:
        got = tb.emulate(q, k, v, dout, mutation=m)
        worst = max((tb.error(n, x, ref[n]) / budget[n], n) for n, x in got.items())
        assert worst[0] >= MARGIN, ("mutation within reach of the budget", m, worst)


def test_emulation_on_bf16_inputs_is_the_oracle():
    """On inputs that are exact in bf16 the emulation only differs from the oracle by the rounding of P and dS to fp32 and then
    to hi + lo (~2^-17): its einsum structure is that of oracle.cca_forward / cca_backward."""
    q, k, v, dout = (tb.bf16(t.double()) for t in _inputs(1, 16, 32, 9, 13, scale=0.5, seed=3))
    ref = tb.reference(q, k, v, dout)
    got = tb.emulate(q, k, v, dout)
    for n in tb.TENSORS:
        assert tb.error(n, got[n], ref[n]) <= 1e-5, n
