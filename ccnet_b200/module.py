"""Drop-in ``CrissCrossAttention`` nn.Module (mirror of cc_attention/functions.py:15-49).

Same constructor, parameter names/shapes/init and forward signature as the reference, so
``networks/ccnet.py:13`` (``from cc_attention import CrissCrossAttention``) and released
checkpoints (``head.cca.*`` keys) work unchanged.  The 1x1 projections stay stock torch
convs (north_star); everything between them and the residual is the CUDA extension.
"""
from __future__ import annotations

from typing import NamedTuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops  # noqa: F401  (torch.ops.cca, which cca* call)

from .functional import (_time_window, cca, cca3d, cca3d_attention, cca3d_step, cca_attention, cca_backward, cca_forward,
                         qkv_gemm_eligible, qkv_project, qkv_project_dgrad, qkv_project_wgrad, qkv_wgrad_eligible,
                         tc3d_eligible, tc_eligible)


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
        ctx.gemm_dtype = outs[0].dtype                                      # fp16 / bf16 under autocast, else x's dtype
        ctx.shape = (B, H, W)
        ctx.wshapes = (wq.shape, wk.shape, wv.shape)
        return tuple(y.view(B, H, W, y.shape[1]).permute(0, 3, 1, 2) for y in outs)   # logical NCHW, channels-last strides

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dq, dk, dv):
        # the backward GEMMs run in the dtype of the forward's (under autocast: the autocast dtype, as the reference's convs do);
        # in-place addmm_ is not autocast, so every operand is brought to that dtype here (no-ops without autocast)
        xm, wq, wk, wv = (t.to(ctx.gemm_dtype) for t in ctx.saved_tensors)
        dq, dk, dv = (g.to(ctx.gemm_dtype) for g in (dq, dk, dv))
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

    def forward(self, x: torch.Tensor, return_attention: bool = False):
        """``return_attention=True`` returns ``(y, attn)``: y exactly as without it, and the step's attention map
        attn[B,H,W,H+W] (float32; the reference's softmax output ``concate``, functions.py:40), differentiable back to x and
        the query / key convs.  The fused kernels never materialise the map, so it costs two more Cq-channel 1x1 convs, a
        second statistics pass and B*H*W*(H+W)*4 bytes; a hook on ``self.softmax`` still does not fire."""
        y = self._step(x)
        if not return_attention:
            return y
        q, k = self.query_conv(x), self.key_conv(x)      # functions.py:29,32
        return y, cca_attention(q, k, self.impl)

    def _step(self, x: torch.Tensor) -> torch.Tensor:
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

    def forward(self, x, return_attention: bool = False):
        """``return_attention=True`` returns ``(out, [attn_1, ..., attn_R])``, the map of every step."""
        out, maps = x, []
        for _ in range(self.recurrence):
            if return_attention:
                out, a = self.cca(out, return_attention=True)
                maps.append(a)
            else:
                out = self.cca(out)
        return (out, maps) if return_attention else out


class RingState(NamedTuple):
    """The stream state of a windowed ``CrissCrossAttention3D.step``: rings of W slots k [B, Cq, W, H, W_img] and
    v [B, C, W, H, W_img] holding the keys and values of the last ``frames`` frames, frame j (oldest first) in slot
    (head + j) % W.  Each step reads the rings and then writes the new frame's k and v into the next free slot or, once the
    rings are full, the oldest frame's slot: the tensors are updated in place and returned in a new ``RingState``."""
    k: torch.Tensor
    v: torch.Tensor
    frames: int
    head: int


class CrissCrossAttention3D(nn.Module):
    """Criss-cross attention over clips x[B, C, T, H, W]: every position attends to the positions that share two of its
    three coordinates (its column, row and time line; T + H + W - 2 keys), y = gamma * cca3d(q(x), k(x), v(x)) + x.
    Parameters mirror ``CrissCrossAttention`` with 1x1x1 Conv3d projections (weights [Cq, C, 1, 1, 1], Cq = C // 8).

    Where the tensor-core path covers the shape, the projections (per pixel) run as GEMMs on the [B*T, C, H, W] frames view
    of channels_last_3d x (a view, no copy) and q, k, v come out channels_last_3d, the layout of those kernels.  Elsewhere
    (other channel counts, T > 32, lines over 896, ``impl="simt"``) the convs are stock Conv3d and the generic kernels run.

    ``causal=True``: frame t attends to the frames before it only (its column and row as before), for models that run on a
    live stream; the parameters and state-dict keys are those of the bidirectional module.  ``step`` then produces one new
    frame from a cache of the past frames' keys and values.

    ``window=W`` (causal only): frame t attends to the frames t - W .. t - 1 only, in ``forward`` as in ``step``, so a model
    trains on clips of any length with the key sets it streams with; ``step`` then keeps a ring of W frames (``RingState``)."""

    def __init__(self, in_dim: int, impl: str = "auto", causal: bool = False, window=None):
        super().__init__()
        window = _time_window(causal, window) or None
        self.query_conv = nn.Conv3d(in_channels=in_dim, out_channels=in_dim // 8, kernel_size=1)
        self.key_conv = nn.Conv3d(in_channels=in_dim, out_channels=in_dim // 8, kernel_size=1)
        self.value_conv = nn.Conv3d(in_channels=in_dim, out_channels=in_dim, kernel_size=1)
        self.gamma = nn.Parameter(torch.zeros(1))
        self.impl = impl
        self.causal = causal
        self.window = window

    def forward(self, x: torch.Tensor, return_attention: bool = False):
        """``return_attention=True`` returns ``(y, attn)``: y exactly as without it, and the attention map
        attn[B,T,H,W,H+W+T] (float32; column, row and time keys, ``ccnet_b200.functional.cca3d_attention_forward``),
        differentiable back to x and the query / key convs.  The fused kernels never materialise the map, so it costs two
        more Cq-channel 1x1x1 convs, a second statistics pass and B*T*H*W*(H+W+T)*4 bytes."""
        y = self._step(x)
        if not return_attention:
            return y
        q, k = self.query_conv(x), self.key_conv(x)
        return y, cca3d_attention(q, k, self.impl, causal=self.causal, window=self.window)

    def _step(self, x: torch.Tensor) -> torch.Tensor:
        if not x.is_cuda:
            raise RuntimeError("ccnet_b200.CrissCrossAttention3D runs on CUDA (H100, sm_90) only")
        B, C, T, H, W = x.shape
        if self.impl != "simt" and tc3d_eligible(B, C // 8, C, T, H, W, x.dtype):
            x = x.contiguous(memory_format=torch.channels_last_3d)
            frames = x.transpose(1, 2).reshape(B * T, C, H, W)             # a channels-last view of the same memory
            q, k, v = _QKVProject.apply(frames, self.query_conv.weight, self.query_conv.bias, self.key_conv.weight,
                                        self.key_conv.bias, self.value_conv.weight, self.value_conv.bias)
            q, k, v = (t.view(B, T, t.shape[1], H, W).transpose(1, 2) for t in (q, k, v))   # channels_last_3d [B, c, T, H, W]
        else:
            q, k, v = self.query_conv(x), self.key_conv(x), self.value_conv(x)
        if q.dtype != v.dtype or k.dtype != v.dtype:       # autocast corner: keep one dtype
            q, k = q.to(v.dtype), k.to(v.dtype)
        return torch.addcmul(x, self.gamma, cca3d(q, k, v, self.impl, causal=self.causal, window=self.window))

    @torch.no_grad()
    def step(self, x_t: torch.Tensor, state=None, max_frames=None):
        """One frame of a stream through the causal module: x_t [B, C, H, W] -> (y_t, state).  ``state`` (None for the first
        frame) holds the keys and values of up to ``max_frames`` previous frames in time order; pass the returned one with the
        next frame.  q, k, v of the frame are the Conv3d projections applied as 1x1 convs, y_t = gamma * out + x_t.

        Frame by frame, ``step`` gives the frames of ``forward(clip)`` while the clip has at most ``max_frames + 1`` frames;
        after that the window slides, and y_t is the last frame of the causal forward on the last ``max_frames + 1`` frames.
        The cost is the 2D op on one frame plus a time pass over the cached frames, instead of the whole window again, plus a
        copy of the cache: each call writes a new one with the new frame's k, v appended.  Inference only (no gradient).
        ``max_frames`` defaults to 31.

        On a module with ``window=W`` the state is a ``RingState`` of W slots, allocated by the first call and then updated
        in place, with no cache copy; frame by frame, ``step`` gives the frames of ``forward(clip)`` for clips of any
        length.  ``max_frames`` must then be left unset or equal W."""
        if not self.causal:
            raise RuntimeError("ccnet_b200.CrissCrossAttention3D.step needs a causal module: CrissCrossAttention3D(in_dim, "
                               "causal=True); a bidirectional frame attends to future frames")
        if self.window is not None and max_frames is not None and max_frames != self.window:
            raise ValueError(f"max_frames of a windowed module is its window ({self.window}), got {max_frames}")
        if not x_t.is_cuda:
            raise RuntimeError("ccnet_b200.CrissCrossAttention3D runs on CUDA (H100, sm_90) only")
        if self.window is not None:
            return self._ring_step(x_t, state)
        max_frames = 31 if max_frames is None else max_frames
        if max_frames < 0:
            raise ValueError("max_frames must be >= 0")
        B, C, H, W = x_t.shape
        S = 0 if state is None else state[0].shape[2]
        tc = self.impl != "simt" and tc3d_eligible(B, C // 8, C, S + 1, H, W, x_t.dtype)
        if tc:
            # channels-last projections: q, k, v come out in the layout of the tensor-core step, and the cache is kept
            # channels_last_3d, so the step does not convert it again
            x_t = x_t.contiguous(memory_format=torch.channels_last)
        q, k, v = (F.conv2d(x_t, conv.weight.squeeze(-1), conv.bias) for conv in (self.query_conv, self.key_conv, self.value_conv))
        if q.dtype != v.dtype or k.dtype != v.dtype:       # autocast corner: keep one dtype
            q, k = q.to(v.dtype), k.to(v.dtype)
        if state is None:
            k_cache, v_cache = k.unsqueeze(2)[:, :, :0], v.unsqueeze(2)[:, :, :0]
        else:
            k_cache, v_cache = state
        out, _ = cca3d_step(q, k, v, k_cache, v_cache, self.impl)
        y = torch.addcmul(x_t, self.gamma.to(out.dtype), out)
        fmt = torch.channels_last_3d if tc else torch.contiguous_format
        return y, (_append_frame(k_cache, k, max_frames, fmt), _append_frame(v_cache, v, max_frames, fmt))

    def _ring_step(self, x_t: torch.Tensor, state):
        B, C, H, W = x_t.shape
        N = self.window
        # the family and layout of the full ring (S = N), for every step of the stream: the rings are never converted
        tc = self.impl != "simt" and tc3d_eligible(B, C // 8, C, N + 1, H, W, x_t.dtype)
        if tc:
            x_t = x_t.contiguous(memory_format=torch.channels_last)
        q, k, v = (F.conv2d(x_t, conv.weight.squeeze(-1), conv.bias) for conv in (self.query_conv, self.key_conv, self.value_conv))
        if q.dtype != v.dtype or k.dtype != v.dtype:       # autocast corner: keep one dtype
            q, k = q.to(v.dtype), k.to(v.dtype)
        if state is None:
            fmt = torch.channels_last_3d if tc else torch.contiguous_format
            ring = lambda t: torch.empty((B, t.shape[1], N, H, W), dtype=t.dtype, device=t.device, memory_format=fmt)
            state = RingState(ring(k), ring(v), 0, 0)
        kr, vr, S, head = state
        out, _ = cca3d_step(q, k, v, kr, vr, "tc" if tc or self.impl == "tc" else "simt", frames=S, head=head)
        y = torch.addcmul(x_t, self.gamma.to(out.dtype), out)
        slot = (head + S) % N                              # the next free slot, or the oldest frame's once the ring is full
        kr[:, :, slot].copy_(k)
        vr[:, :, slot].copy_(v)
        return y, RingState(kr, vr, S + 1, head) if S < N else RingState(kr, vr, N, (head + 1) % N)


def _append_frame(cache: torch.Tensor, x: torch.Tensor, keep: int, fmt) -> torch.Tensor:
    """the last `keep` frames of cat(cache [B,c,S,H,W], x [B,c,H,W]) along time, as one new tensor in memory format `fmt`"""
    n = min(cache.shape[2] + 1, keep)
    out = torch.empty((*x.shape[:2], n, *x.shape[2:]), dtype=x.dtype, device=x.device, memory_format=fmt)
    if n > 1:
        out[:, :, :n - 1].copy_(cache[:, :, cache.shape[2] - (n - 1):])
    if n > 0:
        out[:, :, n - 1].copy_(x)
    return out
