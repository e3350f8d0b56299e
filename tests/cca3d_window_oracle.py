"""fp64 restatement of causal criss-cross attention over clips with a TIME WINDOW, the yardstick of the windowed kernels' and
the ring step's tests.

Pixel u = (b, t, h, w) attends under ONE softmax to its column (self masked), its row and the time keys (b, s, h, w) with
t - W <= s < t.  These are the logits of ``cca3d_causal_oracle.cca3d_causal_logits`` with the time keys s < t - W also set to
-inf; ``window=None`` (every past frame) gives exactly the causal oracle's results (tests/test_cca3d_window_host.py checks
both ties).  The map keeps the layout [B,T,H,W,H+W+T]; time entries outside [t - W, t) are 0.  The gradients are the closed
form of the causal oracle over these logits, checked against autograd.

The ring step: ``cca3d_step`` of the causal oracle on rings [B,c,N,H,W] holding S past frames, frame j in slot (head + j) % N.
"""
from __future__ import annotations

import torch

import cca3d_causal_oracle as OC


def time_mask(T: int, device=None, window=None) -> torch.Tensor:
    """[T, T] bool, True where time key s of query frame t is masked: s >= t, and with a window s < t - window"""
    m = OC.time_mask(T, device)
    return m if window is None else m | torch.ones(T, T, dtype=torch.bool, device=device).tril(-window - 1)


def cca3d_window_logits(q: torch.Tensor, k: torch.Tensor, window=None) -> torch.Tensor:
    """the causal logits with the time keys outside [t - window, t) at -inf"""
    e = OC.cca3d_causal_logits(q, k)
    if window is None:
        return e
    T, H, W = q.shape[2:]
    far = time_mask(T, q.device, window) & ~OC.time_mask(T, q.device)
    return torch.cat([e[..., :H + W], e[..., H + W:].masked_fill(far.view(1, T, 1, 1, T), float("-inf"))], dim=4)


def cca3d_window_attention(q: torch.Tensor, k: torch.Tensor, window=None) -> torch.Tensor:
    """the map [B,T,H,W,H+W+T]: softmax of the windowed logits (masked entries exactly 0)"""
    return torch.softmax(cca3d_window_logits(q, k, window), dim=4)


def cca3d_window_forward(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, window=None):
    """(out[B,C,T,H,W], lse[B,T,H,W])"""
    H, W = q.shape[3:]
    e = cca3d_window_logits(q, k, window)
    return OC._apply(torch.softmax(e, dim=4), v, H, W), torch.logsumexp(e, dim=4)


def cca3d_window_backward(dout: torch.Tensor, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, window=None):
    """(dq, dk, dv) in closed form: P the map, dP = <dout_u, v_j>, delta = <dout, out>, dS = P (dP - delta);
    dq = dS k, dk = dS^T q, dv = P^T dout"""
    H, W = q.shape[3:]
    a = cca3d_window_attention(q, k, window)
    out = OC._apply(a, v, H, W)
    delta = (dout * out).sum(1)                                    # [B,T,H,W]
    dp = torch.cat([torch.einsum("bcthw,bctgw->bthwg", dout, v), torch.einsum("bcthw,bcthg->bthwg", dout, v),
                    torch.einsum("bcthw,bcshw->bthws", dout, v)], dim=4)
    ds = a * (dp - delta.unsqueeze(-1))
    return OC._apply(ds, k, H, W), OC._apply_t(ds, q, H, W), OC._apply_t(a, dout, H, W)


def cca3d_window_attention_backward(dattn: torch.Tensor, q: torch.Tensor, k: torch.Tensor, window=None):
    """(dq, dk) of the map for the upstream gradient dattn: dS = attn (dattn - rho), rho = sum_j attn dattn"""
    H, W = q.shape[3:]
    a = cca3d_window_attention(q, k, window)
    ds = a * (dattn - (a * dattn).sum(-1, keepdim=True))
    return OC._apply(ds, k, H, W), OC._apply_t(ds, q, H, W)


def cca3d_step_ring(q, k, v, k_ring, v_ring, frames=None, head=0):
    """``cca3d_causal_oracle.cca3d_step`` on rings [B,c,N,H,W] holding ``frames`` (None: N) past frames, frame j in slot
    (head + j) % N"""
    N = k_ring.shape[2]
    S = N if frames is None else frames
    idx = torch.tensor([(head + j) % N for j in range(S)], dtype=torch.long)
    return OC.cca3d_step(q, k, v, k_ring.index_select(2, idx), v_ring.index_select(2, idx))


class WindowCrissCrossAttention3DOracle(OC.CausalCrissCrossAttention3DOracle):
    """Module-level restatement of ``ccnet_b200.CrissCrossAttention3D(in_dim, causal=True, window=window)``"""

    def __init__(self, in_dim: int, window=None):
        super().__init__(in_dim)
        self.window = window

    def forward(self, x):
        out, _ = cca3d_window_forward(self.query_conv(x), self.key_conv(x), self.value_conv(x), self.window)
        return self.gamma * out + x


__all__ = ["time_mask", "cca3d_window_logits", "cca3d_window_attention", "cca3d_window_forward", "cca3d_window_backward",
           "cca3d_window_attention_backward", "cca3d_step_ring", "WindowCrissCrossAttention3DOracle"]
