"""``torch.ops.cca.*`` -- the operator ABI SURVEY.md 8(b) specifies, registered with torch's dispatcher:

    torch.ops.cca.forward(q, k, v)                        -> (out, lse)
    torch.ops.cca.backward(dout, q, k, v, out, lse)       -> (dq, dk, dv)
    torch.ops.cca.forward_residual(q, k, v, x, gamma)     -> (y, lse)        y = gamma * out + x  (functions.py:49)
    torch.ops.cca.attention(q, k)                         -> attn            [B,H,W,H+W] fp32 (functions.py:40, `concate`)
    torch.ops.cca.attention_backward(dattn, attn, q, k)   -> (dq, dk)
    torch.ops.cca.forward3d(q, k, v)                      -> (out, lse)      clips [B,C,T,H,W], lse [B,T,H,W]
    torch.ops.cca.backward3d(dout, q, k, v, out, lse)     -> (dq, dk, dv)
    torch.ops.cca.attention3d(q, k)                       -> attn            [B,T,H,W,H+W+T] fp32 (column | row | time)
    torch.ops.cca.attention3d_backward(dattn, attn, q, k) -> (dq, dk)
    torch.ops.cca.forward3d_step(q, k, v, k_cache, v_cache) -> (out, lse)  one new frame of the causal 3D op (inference)

The 3D ops take a trailing ``causal: bool = False`` (CCA_FLAG_CAUSAL: the time keys of frame t are the frames before it) and
``window: int = 0`` (with causal: the frames t - window .. t - 1 only; 0 is every past frame).  ``forward3d_step`` takes
``frames: int = -1, head: int = 0``: the caches are a ring whose slot (head + j) % N holds past frame j (-1: all N slots).

CUDA implementations call the C ABI (ccnet_b200.functional -> libcca_b200.so); FakeTensor ("meta") implementations give
shapes / dtypes / memory formats so that ``torch.compile`` and ``torch.export`` trace through ``networks/ccnet.py`` without a
graph break; autograd is registered on ``forward``, ``forward_residual``, ``attention``, ``forward3d`` and ``attention3d``.  Registration happens through ``torch.library``
(the Python face of TORCH_LIBRARY): the kernels themselves stay behind the torch-free C ABI."""
from __future__ import annotations

from typing import Tuple

import torch
from torch import Tensor

from . import functional as F_


def _out_like(q: Tensor, v: Tensor) -> Tuple[Tensor, Tensor]:
    B, Cq, H, W = q.shape
    fmt = torch.channels_last if F_.tc_eligible(B, Cq, v.shape[1], H, W, q.dtype) else torch.contiguous_format
    return torch.empty(v.shape, dtype=v.dtype, device=v.device).contiguous(memory_format=fmt), \
        torch.empty((B, H, W), dtype=torch.float32, device=q.device)


@torch.library.custom_op("cca::forward", mutates_args=(), device_types="cuda")
def forward(q: Tensor, k: Tensor, v: Tensor) -> Tuple[Tensor, Tensor]:
    return F_.cca_forward(q, k, v)


@forward.register_fake
def _(q, k, v):
    return _out_like(q, v)


@torch.library.custom_op("cca::backward", mutates_args=(), device_types="cuda")
def backward(dout: Tensor, q: Tensor, k: Tensor, v: Tensor, out: Tensor, lse: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
    return F_.cca_backward(dout, q, k, v, out, lse)


@backward.register_fake
def _(dout, q, k, v, out, lse):
    fmt = torch.channels_last if out.is_contiguous(memory_format=torch.channels_last) and out.dim() == 4 else torch.contiguous_format
    mk = lambda t: torch.empty(t.shape, dtype=t.dtype, device=t.device).contiguous(memory_format=fmt)
    return mk(q), mk(k), mk(v)


def _fwd_setup(ctx, inputs, output):
    q, k, v = inputs
    out, lse = output
    ctx.save_for_backward(q, k, v, out, lse)


def _fwd_backward(ctx, dout, dlse):
    q, k, v, out, lse = ctx.saved_tensors
    dq, dk, dv = torch.ops.cca.backward(dout.contiguous(), q, k, v, out, lse)
    return dq, dk, dv


forward.register_autograd(_fwd_backward, setup_context=_fwd_setup)


@torch.library.custom_op("cca::forward_residual", mutates_args=(), device_types="cuda")
def forward_residual(q: Tensor, k: Tensor, v: Tensor, x: Tensor, gamma: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
    """(y, lse, out): y = gamma * out + x; `out` is returned for the backward (delta = <dy, out>)."""
    out, lse = F_.cca_forward(q, k, v)
    return torch.addcmul(x, gamma, out), lse, out


@forward_residual.register_fake
def _(q, k, v, x, gamma):
    out, lse = _out_like(q, v)
    return torch.empty_like(out), lse, out


def _res_setup(ctx, inputs, output):
    q, k, v, x, gamma = inputs
    y, lse, out = output
    ctx.save_for_backward(q, k, v, out, lse, gamma)


def _res_backward(ctx, dy, dlse, dout_unused):
    q, k, v, out, lse, gamma = ctx.saved_tensors
    # the attention backward is linear in dout: run it on dy and scale the (much smaller / equally sized) results by gamma
    dq, dk, dv = torch.ops.cca.backward(dy.contiguous(), q, k, v, out, lse)
    g = gamma.to(dy.dtype)
    return dq * g, dk * g, dv * g, dy, (dy * out).sum().reshape(gamma.shape).to(gamma.dtype)


forward_residual.register_autograd(_res_backward, setup_context=_res_setup)


# ---- the attention map (functions.py:40 `concate`):  attention(q, k) -> attn[B,H,W,H+W] fp32,
#      attention_backward(dattn, attn, q, k) -> (dq, dk)
def _qk_format(q: Tensor) -> torch.memory_format:
    B, Cq, H, W = q.shape
    return torch.channels_last if F_.attention_tc_eligible(B, Cq, H, W, q.dtype) else torch.contiguous_format


@torch.library.custom_op("cca::attention", mutates_args=(), device_types="cuda")
def attention(q: Tensor, k: Tensor, impl: str = "auto") -> Tensor:
    return F_.cca_attention_forward(q, k, impl)


@attention.register_fake
def _(q, k, impl="auto"):
    B, _, H, W = q.shape
    return q.new_empty((B, H, W, H + W), dtype=torch.float32)


@torch.library.custom_op("cca::attention_backward", mutates_args=(), device_types="cuda")
def attention_backward(dattn: Tensor, attn: Tensor, q: Tensor, k: Tensor, impl: str = "auto") -> Tuple[Tensor, Tensor]:
    return F_.cca_attention_backward(dattn, attn, q, k, impl)


@attention_backward.register_fake
def _(dattn, attn, q, k, impl="auto"):
    fmt = torch.channels_last if impl != "simt" and _qk_format(q) == torch.channels_last else torch.contiguous_format
    mk = lambda t: torch.empty(t.shape, dtype=t.dtype, device=t.device).contiguous(memory_format=fmt)
    return mk(q), mk(k)


def _attn_setup(ctx, inputs, output):
    q, k, impl = inputs
    ctx.save_for_backward(q, k, output)
    ctx.impl = impl


def _attn_backward(ctx, dattn):
    q, k, attn = ctx.saved_tensors
    dq, dk = torch.ops.cca.attention_backward(dattn.contiguous(), attn, q, k, ctx.impl)
    return dq, dk, None


attention.register_autograd(_attn_backward, setup_context=_attn_setup)


# ---- criss-cross attention over clips:  forward3d(q, k, v) -> (out, lse[B,T,H,W]),  backward3d(...) -> (dq, dk, dv)
#      (channels_last_3d results on the tensor-core path, contiguous ones on the generic kernels)
@torch.library.custom_op("cca::forward3d", mutates_args=(), device_types="cuda")
def forward3d(q: Tensor, k: Tensor, v: Tensor, causal: bool = False, window: int = 0) -> Tuple[Tensor, Tensor]:
    return F_.cca3d_forward(q, k, v, causal=causal, window=window or None)


@forward3d.register_fake
def _(q, k, v, causal=False, window=0):
    F_._time_window(causal, window or None)
    B, Cq, T, H, W = q.shape
    fmt = torch.channels_last_3d if F_.tc3d_eligible(B, Cq, v.shape[1], T, H, W, q.dtype) else torch.contiguous_format
    return torch.empty(v.shape, dtype=v.dtype, device=v.device).contiguous(memory_format=fmt), \
        torch.empty((B, T, H, W), dtype=torch.float32, device=q.device)


@torch.library.custom_op("cca::backward3d", mutates_args=(), device_types="cuda")
def backward3d(dout: Tensor, q: Tensor, k: Tensor, v: Tensor, out: Tensor, lse: Tensor,
               causal: bool = False, window: int = 0) -> Tuple[Tensor, Tensor, Tensor]:
    return F_.cca3d_backward(dout, q, k, v, out, lse, causal=causal, window=window or None)


@backward3d.register_fake
def _(dout, q, k, v, out, lse, causal=False, window=0):
    fmt = torch.channels_last_3d if out.is_contiguous(memory_format=torch.channels_last_3d) and out.dim() == 5 else torch.contiguous_format
    mk = lambda t: torch.empty(t.shape, dtype=t.dtype, device=t.device).contiguous(memory_format=fmt)
    return mk(q), mk(k), mk(v)


def _fwd3d_setup(ctx, inputs, output):
    q, k, v, causal, window = inputs
    out, lse = output
    ctx.save_for_backward(q, k, v, out, lse)
    ctx.causal = causal
    ctx.window = window


def _fwd3d_backward(ctx, dout, dlse):
    q, k, v, out, lse = ctx.saved_tensors
    dq, dk, dv = torch.ops.cca.backward3d(dout.contiguous(), q, k, v, out, lse, ctx.causal, ctx.window)
    return dq, dk, dv, None, None


forward3d.register_autograd(_fwd3d_backward, setup_context=_fwd3d_setup)


# ---- the attention map over clips:  attention3d(q, k) -> attn[B,T,H,W,H+W+T] fp32,
#      attention3d_backward(dattn, attn, q, k) -> (dq, dk)
@torch.library.custom_op("cca::attention3d", mutates_args=(), device_types="cuda")
def attention3d(q: Tensor, k: Tensor, impl: str = "auto", causal: bool = False, window: int = 0) -> Tensor:
    return F_.cca3d_attention_forward(q, k, impl, causal=causal, window=window or None)


@attention3d.register_fake
def _(q, k, impl="auto", causal=False, window=0):
    F_._time_window(causal, window or None)
    B, _, T, H, W = q.shape
    return q.new_empty((B, T, H, W, H + W + T), dtype=torch.float32)


@torch.library.custom_op("cca::attention3d_backward", mutates_args=(), device_types="cuda")
def attention3d_backward(dattn: Tensor, attn: Tensor, q: Tensor, k: Tensor, impl: str = "auto",
                         causal: bool = False, window: int = 0) -> Tuple[Tensor, Tensor]:
    return F_.cca3d_attention_backward(dattn, attn, q, k, impl, causal=causal, window=window or None)


@attention3d_backward.register_fake
def _(dattn, attn, q, k, impl="auto", causal=False, window=0):
    B, Cq, T, H, W = q.shape
    cl = impl != "simt" and F_.attention3d_tc_eligible(B, Cq, T, H, W, q.dtype)
    fmt = torch.channels_last_3d if cl else torch.contiguous_format
    mk = lambda t: torch.empty(t.shape, dtype=t.dtype, device=t.device).contiguous(memory_format=fmt)
    return mk(q), mk(k)


def _attn3d_setup(ctx, inputs, output):
    q, k, impl, causal, window = inputs
    ctx.save_for_backward(q, k, output)
    ctx.impl = impl
    ctx.causal = causal
    ctx.window = window


def _attn3d_backward(ctx, dattn):
    q, k, attn = ctx.saved_tensors
    dq, dk = torch.ops.cca.attention3d_backward(dattn.contiguous(), attn, q, k, ctx.impl, ctx.causal, ctx.window)
    return dq, dk, None, None, None


attention3d.register_autograd(_attn3d_backward, setup_context=_attn3d_setup)


# ---- the streaming step of the causal 3D op:  forward3d_step(q, k, v, k_cache, v_cache) -> (out[B,C,H,W], lse[B,H,W])
#      (channels-last out on the tensor-core path, contiguous on the generic kernel; no autograd: inference only).  The caches
#      are a ring: frames (-1: all N slots) past frames, frame j in slot (head + j) % N
@torch.library.custom_op("cca::forward3d_step", mutates_args=(), device_types="cuda")
def forward3d_step(q: Tensor, k: Tensor, v: Tensor, k_cache: Tensor, v_cache: Tensor, frames: int = -1,
                   head: int = 0) -> Tuple[Tensor, Tensor]:
    return F_.cca3d_step(q, k, v, k_cache, v_cache, frames=None if frames < 0 else frames, head=head)


@forward3d_step.register_fake
def _(q, k, v, k_cache, v_cache, frames=-1, head=0):
    B, Cq, H, W = q.shape
    S = k_cache.shape[2] if frames < 0 else frames
    cl = F_.tc3d_eligible(B, Cq, v.shape[1], S + 1, H, W, q.dtype)
    fmt = torch.channels_last if cl else torch.contiguous_format
    return torch.empty(v.shape, dtype=v.dtype, device=v.device).contiguous(memory_format=fmt), \
        torch.empty((B, H, W), dtype=torch.float32, device=q.device)
