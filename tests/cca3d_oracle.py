"""fp64 restatement of criss-cross attention over clips (the 3D op), the yardstick of the 3D kernels' tests.

Pixel u = (b, t, h, w) of q, k [B,Cq,T,H,W], v [B,C,T,H,W] attends to three key sets under ONE softmax:
  column {(b, t, g, w)} with g == h masked   (the column branch of the 2D op, cc_attention/functions.py:38)
  row    {(b, t, h, g)}, unmasked            (functions.py:39; the self entry is counted here)
  time   {(b, s, h, w)} with s == t masked
so T + H + W - 2 entries are effective.  At T = 1 the time set is only the masked self and the op is the 2D step on every
frame; with H = 1 it is the 2D step on [B, C, T, W] with T as the column axis.  The reference has no 3D op: the definition
is pinned to it through T = 1 (tests/test_cca3d_host.py against tests/golden/cca_*.npz).
"""
from __future__ import annotations

import torch
import torch.nn as nn


def cca3d_logits(q: torch.Tensor, k: torch.Tensor) -> torch.Tensor:
    """e[b,t,h,w,:] = [column (H) | row (W) | time (T)] logits, -inf at the two masked self entries"""
    B, _, T, H, W = q.shape
    e_h = torch.einsum("bcthw,bctgw->bthwg", q, k)
    e_h = e_h.masked_fill(torch.eye(H, dtype=torch.bool, device=q.device).view(1, 1, H, 1, H), float("-inf"))
    e_w = torch.einsum("bcthw,bcthg->bthwg", q, k)
    e_t = torch.einsum("bcthw,bcshw->bthws", q, k)
    e_t = e_t.masked_fill(torch.eye(T, dtype=torch.bool, device=q.device).view(1, T, 1, 1, T), float("-inf"))
    return torch.cat([e_h, e_w, e_t], dim=4)


def cca3d_forward(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor):
    """(out[B,C,T,H,W], lse[B,T,H,W])"""
    _, _, T, H, W = q.shape
    e = cca3d_logits(q, k)
    a = torch.softmax(e, dim=4)
    a_h, a_w, a_t = a[..., :H], a[..., H:H + W], a[..., H + W:]
    out = (torch.einsum("bthwg,bctgw->bcthw", a_h, v) + torch.einsum("bthwg,bcthg->bcthw", a_w, v)
           + torch.einsum("bthws,bcshw->bcthw", a_t, v))
    return out, torch.logsumexp(e, dim=4)


def cca3d_backward(dout: torch.Tensor, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor):
    """(dq, dk, dv) of ``cca3d_forward`` for the upstream gradient dout (autograd through the einsum restatement)"""
    q, k, v = (t.detach().clone().requires_grad_(True) for t in (q, k, v))
    with torch.enable_grad():
        out, _ = cca3d_forward(q, k, v)
        return torch.autograd.grad(out, (q, k, v), dout)


def cca3d_forward_bruteforce(q, k, v):
    """Loops over every pixel's key set (tiny inputs only)"""
    B, _, T, H, W = q.shape
    out = torch.zeros_like(v)
    lse = torch.zeros((B, T, H, W), dtype=q.dtype)
    for b in range(B):
        for t in range(T):
            for h in range(H):
                for w in range(W):
                    keys = ([(t, g, w) for g in range(H) if g != h] + [(t, h, g) for g in range(W)]
                            + [(s, h, w) for s in range(T) if s != t])
                    e = torch.stack([(q[b, :, t, h, w] * k[b, :, s, g, x]).sum() for s, g, x in keys])
                    a = torch.softmax(e, 0)
                    lse[b, t, h, w] = torch.logsumexp(e, 0)
                    out[b, :, t, h, w] = sum(a[i] * v[b, :, s, g, x] for i, (s, g, x) in enumerate(keys))
    return out, lse


class CrissCrossAttention3DOracle(nn.Module):
    """Module-level restatement of ``ccnet_b200.CrissCrossAttention3D`` with the same parameter names"""

    def __init__(self, in_dim: int):
        super().__init__()
        self.query_conv = nn.Conv3d(in_dim, in_dim // 8, kernel_size=1)
        self.key_conv = nn.Conv3d(in_dim, in_dim // 8, kernel_size=1)
        self.value_conv = nn.Conv3d(in_dim, in_dim, kernel_size=1)
        self.gamma = nn.Parameter(torch.zeros(1))

    def forward(self, x):
        out, _ = cca3d_forward(self.query_conv(x), self.key_conv(x), self.value_conv(x))
        return self.gamma * out + x


def conv3d_state(state2d: dict) -> dict:
    """parameters of the 2D module -> those of the 3D module (1x1 -> 1x1x1 conv weights)"""
    return {n: (p.unsqueeze(-1) if p.dim() == 4 else p) for n, p in state2d.items()}


__all__ = ["cca3d_logits", "cca3d_forward", "cca3d_backward", "cca3d_forward_bruteforce", "CrissCrossAttention3DOracle",
           "conv3d_state"]
