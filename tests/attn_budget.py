"""fp64 oracle of the attention map (cc_attention/functions.py:40, `concate`) and its gradient, an fp64 emulation of the
tensor-core map kernels' arithmetic, and the error budget derived from it.

``attention_map`` = softmax(cat(oracle.cca_logits(q, k))), ``attention_map_backward`` its closed-form gradient w.r.t. q, k.

``emulate`` restates ccnet_b200/csrc/cca_tc_attn.cuh in fp64, the way tests/tc_budget.py restates the other kernels:
  * S = Q K^T as a bf16x3 split for fp32 q, k (16-bit q, k are exact operands); P = exp(S - lse) rounded to fp32.
  * dS = attn (dattn - rho) in fp32, then bf16 hi/lo planes (fp32) or rounded to the 16-bit type; dQ = dS K, dK = dS^T Q;
    16-bit outputs rounded to their type (one rounding per direction and a second one for the add of the two directions).
What it leaves out -- fp32 accumulation order inside the MMAs, exp2f / log2f, the fp32 rounding of S log2e - lse2 -- is
covered by the absolute floor of ``budget``: 2e-5 on the map (lse2 up to ~100 in fp32 costs ~1e-5 relative in P) and on fp32
gradients, two units in the last place of the I/O type on 16-bit gradients.  The generic kernels (impl="simt") compute in
plain fp32 and round 16-bit gradients once, so the same budget bounds them.

Errors are max|got - ref| / max(1, max|ref|) per tensor, as in tests/tc_budget.py.
"""
from __future__ import annotations

import torch

from oracle.cca_oracle import cca_logits
from tc_budget import _mma3, split


def attention_map(q, k):
    """attn[B,H,W,H+W] = softmax over the H+W logits of every pixel, in the dtype of q, k"""
    e_h, e_w = cca_logits(q, k)
    return torch.softmax(torch.cat([e_h, e_w], dim=3), dim=3)


def attention_map_backward(dattn, q, k):
    """(dq, dk) of sum(attention_map(q, k) * dattn), closed form"""
    H = q.shape[2]
    a = attention_map(q, k)
    rho = (a * dattn).sum(-1, keepdim=True)
    ds = a * (dattn - rho)
    ds_h, ds_w = ds[..., :H], ds[..., H:]
    dq = torch.einsum("bhwg,bcgw->bchw", ds_h, k) + torch.einsum("bhwg,bchg->bchw", ds_w, k)
    dk = torch.einsum("bhwg,bchw->bcgw", ds_h, q) + torch.einsum("bhwg,bchw->bchg", ds_w, q)
    return dq, dk


def _round(x, dtype):
    return x.to(dtype).double()


def emulate(q, k, dattn, dtype):
    """the tensor-core kernels' map, dq, dk for q, k of I/O type `dtype` (values already representable in it), in fp64"""
    q, k, dattn = (t.double() for t in (q, k, dattn))
    H = q.shape[2]
    h16 = dtype != torch.float32
    ops = (lambda t: (t, torch.zeros_like(t))) if h16 else split
    sq, sk = ops(q), ops(k)
    eye = torch.eye(H, dtype=torch.bool).view(1, H, 1, H)
    s = torch.cat([_mma3("bchw,bcgw->bhwg", sq, sk).masked_fill(eye, float("-inf")), _mma3("bchw,bchg->bhwg", sq, sk)], dim=3)
    a = _round(torch.exp(s - torch.logsumexp(s, dim=3, keepdim=True)), torch.float32)
    rho = _round((a * dattn).sum(-1, keepdim=True), torch.float32)
    ds = _round(a * (dattn - rho), torch.float32)
    ds = (_round(ds, dtype), torch.zeros_like(ds)) if h16 else split(ds)
    dsh, dsw = (ds[0][..., :H], ds[1][..., :H]), (ds[0][..., H:], ds[1][..., H:])
    r = (lambda t: _round(t, dtype)) if h16 else (lambda t: _round(t, torch.float32))
    dq = r(r(_mma3("bhwg,bcgw->bchw", dsh, sk)) + r(_mma3("bhwg,bchg->bchw", dsw, sk)))
    dk = r(r(_mma3("bhwg,bchw->bcgw", dsh, sq)) + r(_mma3("bhwg,bchw->bchg", dsw, sq)))
    return dict(attn=a, dq=dq, dk=dk)


def reference(q, k, dattn):
    q, k, dattn = (t.double() for t in (q, k, dattn))
    dq, dk = attention_map_backward(dattn, q, k)
    return dict(attn=attention_map(q, k), dq=dq, dk=dk)


def error(got, ref) -> float:
    return (got.detach().cpu().double() - ref).abs().max().item() / max(1.0, ref.abs().max().item())


_ULP = {torch.float32: 0.0, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}


def budget(emulated: dict, ref: dict, dtype) -> dict:
    """per-tensor budget: 4x the emulated kernel's error plus the floor of what the emulation leaves out"""
    floor = dict(attn=2e-5, dq=max(2e-5, 2 * _ULP[dtype]), dk=max(2e-5, 2 * _ULP[dtype]))
    return {n: 4 * error(emulated[n], ref[n]) + floor[n] for n in emulated}


def check(got: dict, ref: dict, bud: dict, what=""):
    errs = {n: error(g, ref[n]) for n, g in got.items()}
    bad = {n: (e, bud[n]) for n, e in errs.items() if not e <= bud[n]}
    assert not bad, (what, "error, budget", bad)
    return errs
