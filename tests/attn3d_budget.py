"""fp64 oracle of the attention map of criss-cross attention over clips, attn[B,T,H,W,H+W+T], and its gradient; an fp64
emulation of the tensor-core kernels' arithmetic (ccnet_b200/csrc/cca_tc_attn3d.cu); the error budget derived from it.

``attention_map3d`` = softmax(cca3d_oracle.cca3d_logits(q, k)), ``attention_map3d_backward`` its closed-form gradient.

``emulate`` restates the kernels the way tests/attn_budget.py restates the 2D map kernels:
  * column and row logits as in the 2D map kernels (bf16x3 split for fp32 q, k; 16-bit q, k are exact operands); time logits
    in plain fp32 FMA from exact inputs (taken as exact); P = exp(S - lse) rounded to fp32, one lse for the whole row.
  * rho and dS = attn (dattn - rho) in fp32; the column / row parts of dq, dk from bf16 hi/lo dS planes (fp32) or dS rounded
    to the 16-bit type, each direction rounded to the I/O type and their sum rounded again; the time part (fp32 dS, fp32 FMA)
    is added onto that and rounded a third time.
  * 16-bit calls that the Python layer runs on the fp32 kernels (functional._upcast: bf16 with T > 1, lines over 112) are
    emulated as fp32 and rounded to the 16-bit type once.
``drop_kstep`` removes one 16-channel k-step from the column part of dq (one MMA of the dq item), the mutation the budget
must catch.  What the emulation leaves out -- fp32 accumulation order, exp2f / log2f, the fp32 rounding of the time logits
-- is covered by the floor of ``attn_budget.budget``.  Errors are max|got - ref| / max(1, max|ref|) per tensor.
"""
from __future__ import annotations

import torch

from attn_budget import _round, budget, check, error  # noqa: F401  (re-exported: one module per budget)
from cca3d_oracle import cca3d_logits
from tc_budget import _mma3, split


def attention_map3d(q, k):
    """attn[B,T,H,W,H+W+T] = softmax over every pixel's column, row and time logits, in the dtype of q, k"""
    return torch.softmax(cca3d_logits(q, k), dim=4)


def _parts(x, H, W):
    return x[..., :H], x[..., H:H + W], x[..., H + W:]


def _dqdk(ds, q, k, H, W):
    """(dq, dk) parts (column, row, time) of dS [B,T,H,W,H+W+T] against exact q, k"""
    dh, dw, dt = _parts(ds, H, W)
    dq = (torch.einsum("bthwg,bctgw->bcthw", dh, k), torch.einsum("bthwg,bcthg->bcthw", dw, k),
          torch.einsum("bthws,bcshw->bcthw", dt, k))
    dk = (torch.einsum("bthwg,bcthw->bctgw", dh, q), torch.einsum("bthwg,bcthw->bcthg", dw, q),
          torch.einsum("bthws,bcthw->bcshw", dt, q))
    return dq, dk


def attention_map3d_backward(dattn, q, k):
    """(dq, dk) of sum(attention_map3d(q, k) * dattn), closed form: dS = attn (dattn - rho), rho = sum_g attn dattn"""
    H, W = q.shape[3], q.shape[4]
    a = attention_map3d(q, k)
    ds = a * (dattn - (a * dattn).sum(-1, keepdim=True))
    dq, dk = _dqdk(ds, q, k, H, W)
    return sum(dq), sum(dk)


def reference(q, k, dattn):
    q, k, dattn = (t.double() for t in (q, k, dattn))
    dq, dk = attention_map3d_backward(dattn, q, k)
    return dict(attn=attention_map3d(q, k), dq=dq, dk=dk)


def emulate(q, k, dattn, dtype, native16: bool = True, drop_kstep: bool = False):
    """the kernels' map, dq, dk for q, k of I/O type `dtype` (values representable in it), in fp64.  native16 = False: a
    16-bit call run on the fp32 kernels and rounded once"""
    q, k, dattn = (t.double() for t in (q, k, dattn))
    B, Cq, T, H, W = q.shape
    h16 = dtype != torch.float32 and native16
    ops = (lambda t: (t, torch.zeros_like(t))) if h16 else split
    sq, sk = ops(q), ops(k)
    e_h = _mma3("bcthw,bctgw->bthwg", sq, sk).masked_fill(torch.eye(H, dtype=torch.bool).view(1, 1, H, 1, H), float("-inf"))
    e_w = _mma3("bcthw,bcthg->bthwg", sq, sk)
    e_t = torch.einsum("bcthw,bcshw->bthws", q, k).masked_fill(torch.eye(T, dtype=torch.bool).view(1, T, 1, 1, T), float("-inf"))
    s = torch.cat([e_h, e_w, e_t], dim=4)
    a = _round(torch.exp(s - torch.logsumexp(s, dim=4, keepdim=True)), torch.float32)
    rho = _round((a * dattn).sum(-1, keepdim=True), torch.float32)
    ds = _round(a * (dattn - rho), torch.float32)
    dh, dw, dt = _parts(ds, H, W)
    pl = (lambda t: (_round(t, dtype), torch.zeros_like(t))) if h16 else split
    kq = (sk[0].clone(), sk[1].clone()) if drop_kstep else sk
    if drop_kstep:
        kq[0][:, Cq - 16:], kq[1][:, Cq - 16:] = 0, 0
    io = dtype if h16 else torch.float32
    r = lambda t: _round(t, io)
    dq = r(r(r(_mma3("bthwg,bctgw->bcthw", pl(dh), kq)) + r(_mma3("bthwg,bcthg->bcthw", pl(dw), sk)))
           + torch.einsum("bthws,bcshw->bcthw", dt, k))
    dk = r(r(r(_mma3("bthwg,bcthw->bctgw", pl(dh), sq)) + r(_mma3("bthwg,bcthw->bcthg", pl(dw), sq)))
           + torch.einsum("bthws,bcthw->bcshw", dt, q))
    if dtype != torch.float32 and not native16:
        dq, dk = _round(dq, dtype), _round(dk, dtype)
    return dict(attn=a, dq=dq, dk=dk)
