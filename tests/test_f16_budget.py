"""CPU test: the fp16 tensor-core error budget (tests/f16_budget.py) sits above the emulated fp16 kernel and below the two
ways a float16 call could silently run in bf16.

  - the budget is at least 2x the emulated floor on every tensor, on every shape;
  - the emulation with its inputs rounded to bf16 (the bf16 kernels on cast tensors) exceeds the budget at least 3x on some
    tensor (lse: the logits lose 3 bits);
  - the emulation with its outputs rounded to bf16 exceeds the budget on some tensor.
The P / dS planes in bf16 are reported, not asserted (see f16_budget.py).  The GPU tests hold the kernels to this budget."""
import pytest
import torch

import f16_budget as fb

SHAPES = [(1, 64, 256, 33, 47), (2, 16, 64, 20, 30), (1, 64, 128, 97, 61), (1, 64, 128, 40, 50)]
SCALES = (0.7, 1.0)


def _inputs(B, Cq, C, H, W, scale, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Cq, H, W, generator=g) * scale
    k = torch.randn(B, Cq, H, W, generator=g) * scale
    v = torch.randn(B, C, H, W, generator=g)
    dout = torch.randn(B, C, H, W, generator=g)
    return tuple(fb.f16(t.double()) for t in (q, k, v, dout))      # what a float16 caller hands the kernels


def _errors(got, ref):
    return {n: fb.error(n, x, ref[n]) for n, x in got.items()}


@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
@pytest.mark.parametrize("scale", SCALES)
def test_f16_budget_separates_the_kernel_from_bf16_roundings(shape, scale):
    q, k, v, dout = _inputs(*shape, scale=scale, seed=sum(shape))
    ref = fb.reference(q, k, v, dout)
    floor = _errors(fb.emulate(q, k, v, dout), ref)
    for n, e in floor.items():
        assert 2.0 * e <= fb.F16_BUDGET[n], ("emulated kernel too close to the budget", n, e, fb.F16_BUDGET[n])
    ratio = {m: max((e / fb.F16_BUDGET[n], n) for n, e in _errors(fb.emulate(q, k, v, dout, mutation=m), ref).items())
             for m in fb.MUTATIONS}
    assert ratio["inputs in bf16"][0] >= 3.0, ratio
    assert ratio["outputs in bf16"][0] > 1.0, ratio
    print(shape, scale, "floor", {n: f"{e:.1e}" for n, e in floor.items()},
          "mutations (worst error / budget)", {m: f"{r:.1f} {n}" for m, (r, n) in ratio.items()})


def test_f16_simt_budget_is_no_tighter_than_the_tensor_core_budget():
    for n in fb.TENSORS:
        assert fb.F16_SIMT[n] >= fb.F16_BUDGET[n], n


def test_emulation_without_roundings_is_the_oracle():
    """With every f16 rounding of the kernel replaced by the identity the emulation is the fp64 oracle: its einsum structure
    is that of oracle.cca_forward / cca_backward."""
    q, k, v, dout = _inputs(1, 16, 32, 9, 13, scale=0.5, seed=3)
    ref = fb.reference(q, k, v, dout)
    saved = fb.f16, fb.fp32
    try:
        fb.f16 = fb.fp32 = lambda x: x
        got = fb.emulate(q, k, v, dout)
    finally:
        fb.f16, fb.fp32 = saved
    for n in fb.TENSORS:
        assert fb.error(n, got[n], ref[n]) <= 1e-12, n
