"""fp64 emulation of the fp16 tensor-core kernels' arithmetic, and the fp16 error budget derived from it.

The fp16 tensor-core kernels (the ``__half`` instantiations of ccnet_b200/csrc/cca_tc_*.cuh) take f16 q, k, v, dout and run
single f16 MMAs with fp32 accumulation: products of two f16 values are exact in fp32, so S = Q K^T, dP = dO V^T and the
products with the P / dS planes are, up to fp32 accumulation, exact.  What rounds is:
  - P = exp(S - lse) and dS = P (dP - delta), each rounded to f16 before it enters an MMA (lse and delta stay fp32);
  - every output.  With one tile per line an output element gets two partial results, one per direction: the column item's
    partial, rounded to f16, is stored; the row item's partial, rounded to f16, is reduce-added onto it by TMA in f16
    arithmetic (the element type of the tensor map), which rounds the sum to f16 once more.
``emulate`` restates that in fp64 with the structure of ``tc_budget.emulate``; the reference is the fp64 oracle on the same
f16 inputs.  fp32 accumulation, exp2f / log2f and the order of the adds are left out: they are orders of magnitude smaller.

``emulate(..., mutation=...)`` replaces one f16 rounding by a bf16 one.  "inputs in bf16" models running the bf16 kernels on
cast tensors, "outputs in bf16" a bf16-typed output map or staging; tests/test_f16_budget.py asserts that the budget catches
both.  "P planes in bf16" and "dS planes in bf16" cannot happen on their own (the other operand of those MMAs is f16, and a
wgmma has one operand type), so they are only reported.

Errors are measured as in tests/tc_budget.py: max|got - ref| / max(1, max|ref|), absolute for lse.
"""
from __future__ import annotations

import torch

from tc_budget import TENSORS, check, error, reference  # noqa: F401  (re-exported: the GPU tests use one module per budget)

# Emulated floor over the shapes of tests/test_f16_budget.py (q, k scale 0.7 - 1.0, Cq <= 64, one tile per line): out 9.5e-4,
# lse 1.9e-6, dq 1.2e-3, dk 1.3e-3, dv 6.8e-4, delta 4e-4 -- set by the f16 rounding of the outputs.  Each budget is >= 2x its
# floor.  Rounding the outputs to bf16 instead costs 2.2x - 3.8x the budget, bf16 inputs cost lse alone ~1000x.
F16_BUDGET = dict(out=2.5e-3, lse=2e-5, dq=3e-3, dk=3e-3, dv=2e-3, delta=1.5e-3)
# the generic (FFMA) kernels on f16 I/O: the same budget for out and lse, 3x for the gradients (their partial sums of the two
# directions are rounded to f16 in memory between the column and the row pass), as for bf16 in test_gpu_tc_edges._budget
F16_SIMT = dict(out=2.5e-3, lse=2e-5, dq=9e-3, dk=9e-3, dv=6e-3, delta=1.5e-3)

MUTATIONS = ("inputs in bf16", "outputs in bf16", "P planes in bf16", "dS planes in bf16")


def f16(x: torch.Tensor) -> torch.Tensor:
    """fp64 tensor -> nearest fp16 (round to nearest even, via fp32), as fp64"""
    return x.float().half().double()


def bf16(x: torch.Tensor) -> torch.Tensor:
    return x.float().to(torch.bfloat16).double()


def fp32(x: torch.Tensor) -> torch.Tensor:
    return x.float().double()


def emulate(q, k, v, dout, mutation=None):
    """The fp16 tensor-core forward and backward on f16-valued inputs (one tile per line), in fp64: dict of out, lse, dq, dk,
    dv, delta."""
    assert mutation is None or mutation in MUTATIONS, mutation
    rin = bf16 if mutation == "inputs in bf16" else f16
    rout = bf16 if mutation == "outputs in bf16" else f16
    rp = bf16 if mutation == "P planes in bf16" else f16
    rds = bf16 if mutation == "dS planes in bf16" else f16

    def two_items(col, row):
        """column item stores its rounded partial, row item reduce-adds its rounded partial (f16 add)"""
        return rout(rout(col) + rout(row))

    q, k, v, dout = (rin(t.double()) for t in (q, k, v, dout))
    H = q.shape[2]
    eye = torch.eye(H, dtype=torch.bool).view(1, H, 1, H)
    s = torch.cat([torch.einsum("bchw,bcgw->bhwg", q, k).masked_fill(eye, float("-inf")),
                   torch.einsum("bchw,bchg->bhwg", q, k)], dim=3)
    lse = fp32(torch.logsumexp(s, dim=3))
    p = rp(fp32(torch.exp(s - lse.unsqueeze(3))))                  # masked entries: exp(-inf) = 0
    pc, pr = p[..., :H], p[..., H:]
    out = two_items(torch.einsum("bhwg,bcgw->bchw", pc, v), torch.einsum("bhwg,bchg->bchw", pr, v))
    # ---- backward: S, P recomputed from the saved lse (the same numbers); delta from the stored f16 out
    delta = fp32((dout * out).sum(1))
    dp = torch.cat([torch.einsum("bchw,bcgw->bhwg", dout, v), torch.einsum("bchw,bchg->bhwg", dout, v)], dim=3)
    dv = two_items(torch.einsum("bhwg,bchw->bcgw", pc, dout), torch.einsum("bhwg,bchw->bchg", pr, dout))
    ds = rds(fp32(p * fp32(dp - delta.unsqueeze(3))))
    dc, dr = ds[..., :H], ds[..., H:]
    dq = two_items(torch.einsum("bhwg,bcgw->bchw", dc, k), torch.einsum("bhwg,bchg->bchw", dr, k))
    dk = two_items(torch.einsum("bhwg,bchw->bcgw", dc, q), torch.einsum("bhwg,bchw->bchg", dr, q))
    return dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv, delta=delta)
