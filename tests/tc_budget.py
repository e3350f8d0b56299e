"""fp64 emulation of the tensor-core kernels' arithmetic, and the fp32 error budget derived from it.

The fp32 tensor-core kernels (ccnet_b200/csrc/cca_tc_*.cu) compute every product as a bf16x3 split: each fp32 operand x is
split into hi = bf16(x) and lo = bf16(x - hi), and a product A B is accumulated as  A_hi B_hi + A_hi B_lo + A_lo B_hi  (the
lo*lo term is dropped).  The attention matrix P = exp(S - lse) and dS = P (dP - delta) are formed in fp32, split the same way
and kept as bf16 hi/lo planes; dS uses the P the planes hold (hi + lo).  ``emulate`` restates that arithmetic in fp64, with the
structure of ``oracle.cca_forward`` / ``oracle.cca_backward``, so its distance from the fp64 oracle is the error a correct
kernel is expected to show.  What it leaves out -- fp32 accumulation inside the MMAs, exp2f / log2f, the order of the adds --
is orders of magnitude smaller.

``mutation`` drops ONE term: the lo part of one operand of one product, or the lo planes of P or dS.  A kernel with such a
bug still looks roughly right; tests/test_tc_budget.py checks that the budgets below sit at least 3x above the emulated
kernel and at least 3x below every such mutation, which is what lets a test at these budgets tell the two apart.

Errors are max|got - ref| / max(1, max|ref|) per tensor (the 1 keeps lines where a gradient vanishes in exact arithmetic,
e.g. a 1x1 map, from dividing by ~0), absolute for lse.
"""
from __future__ import annotations

import torch

TENSORS = ("out", "lse", "dq", "dk", "dv", "delta")

# The error of S = Q K^T is ~2^-17 |q||k| per term, so it grows with the logits' scale and reaches lse directly and every
# other tensor through P.  v, dout ~ N(0, 1) throughout.
# q, k ~ N(0, s^2) with s <= 1, Cq <= 64 (logits of std <= 8).  The emulated floor at s = 1, Cq = 64 is out 7e-5, lse 2.4e-4,
# dq/dk 5e-5, dv 3e-5, delta 4e-5; at s = 0.7 about a third of that.  A single dropped term costs >= 1.2e-3.
FP32_BUDGET = dict(out=2e-4, lse=8e-4, dq=1.5e-4, dk=1.5e-4, dv=1e-4, delta=1.5e-4)
# q, k ~ N(0, 1.5^2), Cq = 64 (logits of std ~18, near one-hot attention).  Floor: out, dq, dk, delta up to 1.2e-4, lse 4.8e-4,
# dv 4e-5.  lse keeps the 1e-3 the forward stress test has always used: it is only 2x its floor, which the arithmetic
# leaves no room to improve (lse is the largest logit, ~90 here, and carries that logit's whole error).
FP32_PEAKED_BUDGET = dict(out=4e-4, lse=1e-3, dq=4e-4, dk=4e-4, dv=1.5e-4, delta=4e-4)
# plain fp32 FMA (the generic kernels, impl="simt"): lse absolute, the rest relative as above
FP32_SIMT = dict(out=2e-5, lse=2e-5, dq=2e-5, dk=2e-5, dv=2e-5, delta=2e-5)

# name -> (product, operand whose lo part is dropped) or (planes, "hi-only")
MUTATIONS = {
    "S=QK^T without Q_lo": ("S", 0), "S=QK^T without K_lo": ("S", 1),
    "O=PV without P_lo": ("O", 0), "O=PV without V_lo": ("O", 1),
    "dP=dO V^T without dO_lo": ("dP", 0), "dP=dO V^T without V_lo": ("dP", 1),
    "dV=P^T dO without P_lo": ("dV", 0), "dV=P^T dO without dO_lo": ("dV", 1),
    "dQ=dS K without dS_lo": ("dQ", 0), "dQ=dS K without K_lo": ("dQ", 1),
    "dK=dS^T Q without dS_lo": ("dK", 0), "dK=dS^T Q without Q_lo": ("dK", 1),
    "P planes hi-only": ("P", None), "dS planes hi-only": ("dS", None),
}


def bf16(x: torch.Tensor) -> torch.Tensor:
    """fp64 tensor of fp32 values -> the nearest bf16 (round to nearest even), as fp64"""
    return x.float().to(torch.bfloat16).double()


def fp32(x: torch.Tensor) -> torch.Tensor:
    return x.float().double()


def split(x: torch.Tensor, keep_lo: bool = True):
    """(hi, lo) of an fp32 value; x - hi is exact in fp32, so lo = bf16(x - hi)"""
    hi = bf16(x)
    return hi, (bf16(x - hi) if keep_lo else torch.zeros_like(x))


def _mma3(eq, a, b, drop=None):
    """bf16x3 product of two (hi, lo) operands, exact (fp64) accumulation; drop = 0 / 1: that operand's lo term is missing"""
    (ah, al), (bh, bl) = a, b
    r = torch.einsum(eq, ah, bh)
    if drop != 1:
        r = r + torch.einsum(eq, ah, bl)
    if drop != 0:
        r = r + torch.einsum(eq, al, bh)
    return r


def emulate(q, k, v, dout, mutation=None):
    """The fp32 tensor-core forward and backward on fp32-valued inputs, in fp64: dict of out, lse, dq, dk, dv, delta."""
    prod, which = MUTATIONS[mutation] if mutation else (None, None)
    d = lambda name: which if prod == name else None
    q, k, v, dout = (t.double() for t in (q, k, v, dout))
    H = q.shape[2]
    sq, sk, sv, sdo = split(q), split(k), split(v), split(dout)
    # ---- forward: statistics + values
    eye = torch.eye(H, dtype=torch.bool).view(1, H, 1, H)
    s = torch.cat([_mma3("bchw,bcgw->bhwg", sq, sk, d("S")).masked_fill(eye, float("-inf")),
                   _mma3("bchw,bchg->bhwg", sq, sk, d("S"))], dim=3)
    lse = fp32(torch.logsumexp(s, dim=3))
    p = fp32(torch.exp(s - lse.unsqueeze(3)))                      # masked entries: exp(-inf) = 0
    ph, pw = split(p[..., :H]), split(p[..., H:])
    out = fp32(_mma3("bhwg,bcgw->bchw", ph, sv, d("O")) + _mma3("bhwg,bchg->bchw", pw, sv, d("O")))
    # ---- backward (recomputes S, P from the saved lse: the same numbers)
    keep = prod != "P"
    ph, pw = split(p[..., :H], keep), split(p[..., H:], keep)
    dp = torch.cat([_mma3("bchw,bcgw->bhwg", sdo, sv, d("dP")), _mma3("bchw,bchg->bhwg", sdo, sv, d("dP"))], dim=3)
    delta = fp32((dout * out).sum(1))
    dv = fp32(_mma3("bhwg,bchw->bcgw", ph, sdo, d("dV")) + _mma3("bhwg,bchw->bchg", pw, sdo, d("dV")))
    pr = torch.cat([ph[0] + ph[1], pw[0] + pw[1]], dim=3)          # the P the planes hold
    ds = fp32(pr * fp32(dp - delta.unsqueeze(3)))
    keep = prod != "dS"
    dsh, dsw = split(ds[..., :H], keep), split(ds[..., H:], keep)
    dq = fp32(_mma3("bhwg,bcgw->bchw", dsh, sk, d("dQ")) + _mma3("bhwg,bchg->bchw", dsw, sk, d("dQ")))
    dk = fp32(_mma3("bhwg,bchw->bcgw", dsh, sq, d("dK")) + _mma3("bhwg,bchw->bchg", dsw, sq, d("dK")))
    return dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv, delta=delta)


def reference(q, k, v, dout):
    """fp64 oracle of the same tensors (delta = <dout, out> per pixel, the tensor-core backward's by-product)"""
    from oracle import cca_oracle as O
    q, k, v, dout = (t.double() for t in (q, k, v, dout))
    out, lse = O.cca_forward(q, k, v)
    dq, dk, dv = O.cca_backward(dout, q, k, v)
    return dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv, delta=(dout * out).sum(1))


def error(name: str, got: torch.Tensor, ref: torch.Tensor) -> float:
    """the error measure the budgets are stated in"""
    e = (got.detach().cpu().double() - ref).abs().max().item()
    return e if name == "lse" else e / max(1.0, ref.abs().max().item())


def check(got: dict, ref: dict, budget: dict, what=""):
    """assert every tensor of `got` (any subset of TENSORS) is within `budget` of `ref`; returns {name: error}"""
    errs = {n: error(n, g, ref[n]) for n, g in got.items()}
    bad = {n: (e, budget[n]) for n, e in errs.items() if not e <= budget[n]}
    assert not bad, (what, "error, budget", bad)
    return errs
