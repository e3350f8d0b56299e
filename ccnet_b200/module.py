"""Drop-in ``CrissCrossAttention`` nn.Module (mirror of cc_attention/functions.py:15-49).

Same constructor, parameter names/shapes/init and forward signature as the reference, so
``networks/ccnet.py:13`` (``from cc_attention import CrissCrossAttention``) and released
checkpoints (``head.cca.*`` keys) work unchanged.  The 1x1 projections stay stock torch
convs (north_star); everything between them and the residual is the CUDA extension.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from .functional import (cca, cca_backward, cca_forward, qkv_gemm_eligible, qkv_project, qkv_project_dgrad,
                         qkv_project_wgrad, qkv_wgrad_eligible, tc_eligible)


class _QKVProject(torch.autograd.Function):
    """The three 1x1 convs of functions.py:29,32,35 on a channels-last tensor, as dense GEMMs on its [pixels, C] view
    (cuBLAS; same parameters and fp32 maths as ``conv(x)``).  The outputs are channels-last q, k, v -- exactly the layout
    the tensor-core kernels consume.  One autograd node instead of three so that the input gradient is accumulated inside
    the GEMMs (beta = 1) rather than by two extra elementwise passes over [pixels, C]."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda")
    def forward(ctx, x_cl, wq, bq, wk, bk, wv, bv):
        B, C, H, W = x_cl.shape
        xm = x_cl.permute(0, 2, 3, 1).reshape(B * H * W, C)                # a view: channels-last memory is [pixels, C]
        ws = [w.view(w.shape[0], C) for w in (wq, wk, wv)]
        outs = [torch.addmm(b, xm, w.t()) for w, b in zip(ws, (bq, bk, bv))]
        ctx.save_for_backward(xm, *ws)
        ctx.shape = (B, H, W)
        ctx.wshapes = (wq.shape, wk.shape, wv.shape)
        return tuple(y.view(B, H, W, y.shape[1]).permute(0, 3, 1, 2) for y in outs)   # logical NCHW, channels-last strides

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dq, dk, dv):
        xm, wq, wk, wv = ctx.saved_tensors
        dq, dk, dv = (g.to(xm.dtype) for g in (dq, dk, dv))                # autocast may hand back reduced-precision grads
        B, H, W = ctx.shape
        C = xm.shape[1]
        gs = [g.permute(0, 2, 3, 1).reshape(B * H * W, g.shape[1]) for g in (dq, dk, dv)]   # views of channels-last grads
        dx = torch.mm(gs[2], wv)
        dx.addmm_(gs[0], wq)
        dx.addmm_(gs[1], wk)
        dws = [torch.mm(g.t(), xm).view(shp) for g, shp in zip(gs, ctx.wshapes)]
        dbs = [g.sum(0) for g in gs]
        dx = dx.view(B, H, W, C).permute(0, 3, 1, 2)
        return dx, dws[0], dbs[0], dws[1], dbs[1], dws[2], dbs[2]


class _FusedCCAStep(torch.autograd.Function):
    """y = gamma * cca(q(x), k(x), v(x)) + x  -- functions.py:29-49 as ONE autograd node on channels-last fp32 tensors:
    projections and their input gradient on the hand-written wgmma GEMMs, the attention on the wgmma item kernels.

    The backward exploits that the attention backward is linear in dout: it runs on dy itself and the factor gamma is applied
    to the three small weight matrices of the input-gradient GEMM (and to the weight gradients) instead of scaling the [B,C,H,W]
    tensor dout = gamma * dy in an extra pass; dgamma = <dy, o> (functions.py:49)."""

    @staticmethod
    def forward(ctx, x, wq, bq, wk, bk, wv, bv, gamma):
        B, C, H, W = x.shape
        wq2, wk2, wv2 = (w.reshape(w.shape[0], C) for w in (wq, wk, wv))
        q, k, v = qkv_project(x, wq2, bq, wk2, bk, wv2, bv)
        o, lse = cca_forward(q, k, v, "tc")
        ctx.save_for_backward(x, q, k, v, o, lse, wq2, wk2, wv2, gamma)
        ctx.wshapes = (wq.shape, wk.shape, wv.shape)
        return torch.addcmul(x, gamma, o)                                   # functions.py:49

    @staticmethod
    def backward(ctx, dy):
        x, q, k, v, o, lse, wq, wk, wv, gamma = ctx.saved_tensors
        B, C, H, W = x.shape
        dy = dy.contiguous(memory_format=torch.channels_last)
        dq, dk, dv, delta = cca_backward(dy, q, k, v, o, lse, "tc", want_delta=True)   # for dout = dy (gamma pending)
        g = gamma.detach().to(dy.dtype).contiguous()
        dx = qkv_project_dgrad(dq, dk, dv, wq, wk, wv, scale=g)             # gamma rides on the packed weights
        dx += dy                                                            # the residual branch
        dgamma = delta.sum().reshape(1)                                     # <dy, o>: the kernel's per-pixel delta, summed
        if qkv_wgrad_eligible(C, q.shape[1]):
            dwq, dbq, dwk, dbk, dwv, dbv = qkv_project_wgrad(x, dq, dk, dv, scale=g)
            shp = ctx.wshapes
            return dx, dwq.view(shp[0]), dbq, dwk.view(shp[1]), dbk, dwv.view(shp[2]), dbv, dgamma
        xm = x.permute(0, 2, 3, 1).reshape(B * H * W, C)
        grads = []
        for t, shp in zip((dq, dk, dv), ctx.wshapes):
            gm = t.permute(0, 2, 3, 1).reshape(B * H * W, t.shape[1])
            grads.append((torch.mm(gm.t(), xm).mul_(g).view(shp), gm.sum(0).mul_(g)))
        return dx, grads[0][0], grads[0][1], grads[1][0], grads[1][1], grads[2][0], grads[2][1], dgamma


class CrissCrossAttention(nn.Module):
    """Criss-Cross Attention Module (Hopper-native operator behind the reference surface)."""

    def __init__(self, in_dim: int, impl: str = "auto"):
        super().__init__()
        self.query_conv = nn.Conv2d(in_channels=in_dim, out_channels=in_dim // 8, kernel_size=1)  # functions.py:19
        self.key_conv = nn.Conv2d(in_channels=in_dim, out_channels=in_dim // 8, kernel_size=1)    # functions.py:20
        self.value_conv = nn.Conv2d(in_channels=in_dim, out_channels=in_dim, kernel_size=1)       # functions.py:21
        self.softmax = nn.Softmax(dim=3)      # kept for attribute parity (functions.py:22); fused in the kernel
        self.INF = None                       # functions.py:23 -- the mask is a predicate inside the kernel
        self.gamma = nn.Parameter(torch.zeros(1))                                                  # functions.py:24
        self.impl = impl

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not x.is_cuda:
            raise RuntimeError("ccnet_b200.CrissCrossAttention runs on CUDA (H100, sm_90) only; "
                               "the CPU restatement lives in oracle/ and is test-only")
        B, C, H, W = x.shape
        if (self.impl != "simt" and tc_eligible(B, C // 8, C, H, W, x.dtype) and qkv_gemm_eligible(x, C // 8)
                and not torch.is_autocast_enabled()):
            # everything on hand-written sm_90a kernels: projection GEMMs + attention + their backward, one autograd node
            x = x.contiguous(memory_format=torch.channels_last)
            return _FusedCCAStep.apply(x, self.query_conv.weight, self.query_conv.bias, self.key_conv.weight,
                                       self.key_conv.bias, self.value_conv.weight, self.value_conv.bias, self.gamma)
        if self.impl != "simt" and tc_eligible(B, C // 8, C, H, W, x.dtype):
            # tensor-core kernels are channels-last; converting x once (a no-op inside a channels_last network) lets
            # the three 1x1 projections run as plain GEMMs that emit channels-last q/k/v directly
            x = x.contiguous(memory_format=torch.channels_last)
            q, k, v = _QKVProject.apply(x, self.query_conv.weight, self.query_conv.bias,      # functions.py:29
                                        self.key_conv.weight, self.key_conv.bias,          # functions.py:32
                                        self.value_conv.weight, self.value_conv.bias)      # functions.py:35
        else:
            q = self.query_conv(x)            # functions.py:29
            k = self.key_conv(x)              # functions.py:32
            v = self.value_conv(x)            # functions.py:35
        if q.dtype != v.dtype or k.dtype != v.dtype:       # autocast corner: keep one dtype
            q, k = q.to(v.dtype), k.to(v.dtype)
        o = cca(q, k, v, self.impl)           # functions.py:30-47 fused
        return torch.addcmul(x, self.gamma, o)          # gamma * o + x in one pass (functions.py:49)


class RCCA(nn.Module):
    """The recurrence of networks/ccnet.py:116-119: the same CCA module applied R times."""

    def __init__(self, in_dim: int, recurrence: int = 2, impl: str = "auto"):
        super().__init__()
        self.cca = CrissCrossAttention(in_dim, impl)
        self.recurrence = recurrence

    def forward(self, x):
        out = x
        for _ in range(self.recurrence):
            out = self.cca(out)
        return out
