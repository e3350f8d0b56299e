"""fp64 restatement of CAUSAL criss-cross attention over clips (CCA_FLAG_CAUSAL), the yardstick of the causal kernels' tests.

Pixel u = (b, t, h, w) attends under ONE softmax to
  column {(b, t, g, w)} with g == h masked   (as in tests/cca3d_oracle.py)
  row    {(b, t, h, g)}, unmasked
  time   {(b, s, h, w)} with s < t only
Frame 0 has no time key: its row is the 2D op's.  The logits are those of ``cca3d_oracle.cca3d_logits`` with the time keys
s > t also set to -inf (tests/test_cca3d_causal_host.py checks both ties to that oracle).  The map keeps the layout
[B,T,H,W,H+W+T]; its time entries s >= t are 0.  The gradients are written in closed form (dS = P (dP - delta)), checked
against autograd on ``cca3d_causal_forward``.

The streaming step: frame S of the causal forward on the clip whose frames 0..S-1 have keys k_cache, values v_cache and whose
frame S has q, k, v (the past queries do not enter).
"""
from __future__ import annotations

import torch

import cca3d_oracle as O3


def time_mask(T: int, device=None) -> torch.Tensor:
    """[T, T] bool, True where time key s of query frame t is masked (s >= t)"""
    return torch.ones(T, T, dtype=torch.bool, device=device).triu()


def cca3d_causal_logits(q: torch.Tensor, k: torch.Tensor) -> torch.Tensor:
    """e[b,t,h,w,:] = [column (H) | row (W) | time (T)] logits, -inf at the column's self entry and at time keys s >= t"""
    B, _, T, H, W = q.shape
    e_h = torch.einsum("bcthw,bctgw->bthwg", q, k)
    e_h = e_h.masked_fill(torch.eye(H, dtype=torch.bool, device=q.device).view(1, 1, H, 1, H), float("-inf"))
    e_w = torch.einsum("bcthw,bcthg->bthwg", q, k)
    e_t = torch.einsum("bcthw,bcshw->bthws", q, k)
    e_t = e_t.masked_fill(time_mask(T, q.device).view(1, T, 1, 1, T), float("-inf"))
    return torch.cat([e_h, e_w, e_t], dim=4)


def cca3d_causal_attention(q: torch.Tensor, k: torch.Tensor) -> torch.Tensor:
    """the map [B,T,H,W,H+W+T]: softmax of the causal logits (masked entries exactly 0)"""
    return torch.softmax(cca3d_causal_logits(q, k), dim=4)


def _apply(a: torch.Tensor, x: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """sum over the row of a [B,T,H,W,H+W+T] of a * (the key's x), x [B,C,T,H,W]"""
    return (torch.einsum("bthwg,bctgw->bcthw", a[..., :H], x) + torch.einsum("bthwg,bcthg->bcthw", a[..., H:H + W], x)
            + torch.einsum("bthws,bcshw->bcthw", a[..., H + W:], x))


def _apply_t(a: torch.Tensor, y: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """the transpose of ``_apply``: key pixel j collects sum over the queries u of a[u, entry of j] * y_u"""
    return (torch.einsum("bthwg,bcthw->bctgw", a[..., :H], y) + torch.einsum("bthwg,bcthw->bcthg", a[..., H:H + W], y)
            + torch.einsum("bthws,bcthw->bcshw", a[..., H + W:], y))


def cca3d_causal_forward(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor):
    """(out[B,C,T,H,W], lse[B,T,H,W])"""
    _, _, _, H, W = q.shape
    e = cca3d_causal_logits(q, k)
    return _apply(torch.softmax(e, dim=4), v, H, W), torch.logsumexp(e, dim=4)


def cca3d_causal_backward(dout: torch.Tensor, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor):
    """(dq, dk, dv) in closed form: P the map, dP = <dout_u, v_j>, delta = <dout, out>, dS = P (dP - delta);
    dq = dS k, dk = dS^T q, dv = P^T dout"""
    _, _, _, H, W = q.shape
    a = cca3d_causal_attention(q, k)
    out = _apply(a, v, H, W)
    delta = (dout * out).sum(1)                                    # [B,T,H,W]
    dp = torch.cat([torch.einsum("bcthw,bctgw->bthwg", dout, v), torch.einsum("bcthw,bcthg->bthwg", dout, v),
                    torch.einsum("bcthw,bcshw->bthws", dout, v)], dim=4)
    ds = a * (dp - delta.unsqueeze(-1))
    return _apply(ds, k, H, W), _apply_t(ds, q, H, W), _apply_t(a, dout, H, W)


def cca3d_causal_attention_backward(dattn: torch.Tensor, q: torch.Tensor, k: torch.Tensor):
    """(dq, dk) of the map for the upstream gradient dattn: dS = attn (dattn - rho), rho = sum_j attn dattn"""
    _, _, _, H, W = q.shape
    a = cca3d_causal_attention(q, k)
    ds = a * (dattn - (a * dattn).sum(-1, keepdim=True))
    return _apply(ds, k, H, W), _apply_t(ds, q, H, W)


def cca3d_step(q, k, v, k_cache, v_cache):
    """(out[B,C,H,W], lse[B,H,W]) of the new frame: frame S of the causal forward on the clip cat(cache, frame).  The past
    frames' queries do not enter; any value stands in for them."""
    kk = torch.cat([k_cache, k.unsqueeze(2)], 2)
    vv = torch.cat([v_cache, v.unsqueeze(2)], 2)
    qq = torch.zeros_like(kk)
    qq[:, :, -1] = q
    out, lse = cca3d_causal_forward(qq, kk, vv)
    return out[:, :, -1], lse[:, -1]


class CausalCrissCrossAttention3DOracle(O3.CrissCrossAttention3DOracle):
    """Module-level restatement of ``ccnet_b200.CrissCrossAttention3D(in_dim, causal=True)``"""

    def forward(self, x):
        out, _ = cca3d_causal_forward(self.query_conv(x), self.key_conv(x), self.value_conv(x))
        return self.gamma * out + x


__all__ = ["time_mask", "cca3d_causal_logits", "cca3d_causal_attention", "cca3d_causal_forward", "cca3d_causal_backward",
           "cca3d_causal_attention_backward", "cca3d_step", "CausalCrissCrossAttention3DOracle"]
