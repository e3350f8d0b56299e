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

After the tensors come defaulted arguments (new ones are appended, so positional calls keep their meaning):

    forward, backward, attention, attention_backward      impl="auto", deterministic=None
    forward3d, backward3d                                 causal=False, window=0, impl="auto", deterministic=None
    attention3d, attention3d_backward                     impl="auto", causal=False, window=0, deterministic=None
    forward3d_step                                        frames=-1, head=0

``impl`` ("auto" | "tc" | "simt") and ``deterministic`` (None follows ``torch.are_deterministic_algorithms_enabled()``) mean
what they mean for ``ccnet_b200.functional.cca_forward``.  ``causal`` (CCA_FLAG_CAUSAL): the time keys of frame t are the
frames before it; ``window`` (with causal): the frames t - window .. t - 1 only, 0 is every past frame.  The caches of
``forward3d_step`` are a ring whose slot (head + j) % N holds past frame j (frames=-1: all N slots).

CUDA implementations call the C ABI (ccnet_b200.functional -> libcca_b200.so); FakeTensor ("meta") implementations give
shapes / dtypes / memory formats, planned by ``functional._plan`` like the real calls, so that ``torch.compile`` and
``torch.export`` trace through ``networks/ccnet.py`` without a graph break.  Autograd is registered on ``forward``,
``forward_residual``, ``attention``, ``forward3d`` and ``attention3d``; it is the autograd of the differentiable entry
points ``ccnet_b200.cca``, ``cca_attention``, ``cca3d`` and ``cca3d_attention``, which call these ops.  Registration happens
through ``torch.library`` (the Python face of TORCH_LIBRARY): the kernels themselves stay behind the torch-free C ABI."""
from __future__ import annotations

from typing import Optional, Tuple

import torch
from torch import Tensor

from . import capi
from . import functional as F_


def _format(impl: str, covered, q: Tensor, v: Optional[Tensor] = None) -> torch.memory_format:
    """the memory format of a fake's results: the real call's, by its coverage query (impl="tc" off it raises)"""
    return F_._plan(impl, False, covered, q, v)[2]


def _out_lse(fmt, q: Tensor, v: Tensor) -> Tuple[Tensor, Tensor]:
    """out like v in ``fmt`` and lse float32 [B, *q.shape[2:]]"""
    return torch.empty_like(v, memory_format=fmt), q.new_empty((q.shape[0], *q.shape[2:]), dtype=torch.float32)


@torch.library.custom_op("cca::forward", mutates_args=(), device_types="cuda")
def forward(q: Tensor, k: Tensor, v: Tensor, impl: str = "auto",
            deterministic: Optional[bool] = None) -> Tuple[Tensor, Tensor]:
    return F_.cca_forward(q, k, v, impl, deterministic)


@forward.register_fake
def _(q, k, v, impl="auto", deterministic=None):
    return _out_lse(_format(impl, F_._covered(capi.CCA_WS_FORWARD, q, v), q, v), q, v)


@torch.library.custom_op("cca::backward", mutates_args=(), device_types="cuda")
def backward(dout: Tensor, q: Tensor, k: Tensor, v: Tensor, out: Tensor, lse: Tensor, impl: str = "auto",
             deterministic: Optional[bool] = None) -> Tuple[Tensor, Tensor, Tensor]:
    return F_.cca_backward(dout, q, k, v, out, lse, impl, deterministic=deterministic)


@backward.register_fake
def _(dout, q, k, v, out, lse, impl="auto", deterministic=None):
    fmt = _format(impl, F_._covered(capi.CCA_WS_BACKWARD, q, v), q, v)
    return tuple(torch.empty_like(t, memory_format=fmt) for t in (q, k, v))


@torch.library.custom_op("cca::forward_residual", mutates_args=(), device_types="cuda")
def forward_residual(q: Tensor, k: Tensor, v: Tensor, x: Tensor, gamma: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
    """(y, lse, out): y = gamma * out + x; `out` is returned for the backward (delta = <dy, out>)."""
    out, lse = F_.cca_forward(q, k, v)
    return torch.addcmul(x, gamma, out), lse, out


@forward_residual.register_fake
def _(q, k, v, x, gamma):
    out, lse = _out_lse(_format("auto", F_._covered(capi.CCA_WS_FORWARD, q, v), q, v), q, v)
    return torch.addcmul(x, gamma, out), lse, out                  # (y takes its strides from x and out, as the real one)


def _res_setup(ctx, inputs, output):
    q, k, v, x, gamma = inputs
    y, lse, out = output
    ctx.save_for_backward(q, k, v, out, lse, gamma)


def _res_backward(ctx, dy, dlse, dout_unused):
    q, k, v, out, lse, gamma = ctx.saved_tensors
    # the attention backward is linear in dout: run it on dy and scale the (much smaller / equally sized) results by gamma
    dq, dk, dv = torch.ops.cca.backward(dy, q, k, v, out, lse)
    g = gamma.to(dy.dtype)
    return dq * g, dk * g, dv * g, dy, (dy * out).sum().reshape(gamma.shape).to(gamma.dtype)


forward_residual.register_autograd(_res_backward, setup_context=_res_setup)


# ---- the attention map (functions.py:40 `concate`):  attention(q, k) -> attn[B,H,W,H+W] fp32,
#      attention_backward(dattn, attn, q, k) -> (dq, dk)
@torch.library.custom_op("cca::attention", mutates_args=(), device_types="cuda")
def attention(q: Tensor, k: Tensor, impl: str = "auto", deterministic: Optional[bool] = None) -> Tensor:
    return F_.cca_attention_forward(q, k, impl, deterministic)


@attention.register_fake
def _(q, k, impl="auto", deterministic=None):
    _format(impl, F_._attention_covered(q), q)
    B, _, H, W = q.shape
    return q.new_empty((B, H, W, H + W), dtype=torch.float32)


@torch.library.custom_op("cca::attention_backward", mutates_args=(), device_types="cuda")
def attention_backward(dattn: Tensor, attn: Tensor, q: Tensor, k: Tensor, impl: str = "auto",
                       deterministic: Optional[bool] = None) -> Tuple[Tensor, Tensor]:
    return F_.cca_attention_backward(dattn, attn, q, k, impl, deterministic)


@attention_backward.register_fake
def _(dattn, attn, q, k, impl="auto", deterministic=None):
    fmt = _format(impl, F_._attention_covered(q), q)
    return torch.empty_like(q, memory_format=fmt), torch.empty_like(k, memory_format=fmt)


# ---- criss-cross attention over clips:  forward3d(q, k, v) -> (out, lse[B,T,H,W]),  backward3d(...) -> (dq, dk, dv)
#      (channels_last_3d results on the tensor-core path, contiguous ones on the generic kernels)
@torch.library.custom_op("cca::forward3d", mutates_args=(), device_types="cuda")
def forward3d(q: Tensor, k: Tensor, v: Tensor, causal: bool = False, window: int = 0, impl: str = "auto",
              deterministic: Optional[bool] = None) -> Tuple[Tensor, Tensor]:
    return F_.cca3d_forward(q, k, v, impl, deterministic, causal, window or None)


@forward3d.register_fake
def _(q, k, v, causal=False, window=0, impl="auto", deterministic=None):
    F_._time_window(causal, window or None)
    return _out_lse(_format(impl, F_._covered3d(capi.CCA_WS_FORWARD, q, v, q.shape[2]), q, v), q, v)


@torch.library.custom_op("cca::backward3d", mutates_args=(), device_types="cuda")
def backward3d(dout: Tensor, q: Tensor, k: Tensor, v: Tensor, out: Tensor, lse: Tensor, causal: bool = False,
               window: int = 0, impl: str = "auto", deterministic: Optional[bool] = None) -> Tuple[Tensor, Tensor, Tensor]:
    return F_.cca3d_backward(dout, q, k, v, out, lse, impl, deterministic, causal, window or None)


@backward3d.register_fake
def _(dout, q, k, v, out, lse, causal=False, window=0, impl="auto", deterministic=None):
    fmt = _format(impl, F_._covered3d(capi.CCA_WS_BACKWARD, q, v, q.shape[2]), q, v)
    return tuple(torch.empty_like(t, memory_format=fmt) for t in (q, k, v))


# ---- the attention map over clips:  attention3d(q, k) -> attn[B,T,H,W,H+W+T] fp32,
#      attention3d_backward(dattn, attn, q, k) -> (dq, dk)
@torch.library.custom_op("cca::attention3d", mutates_args=(), device_types="cuda")
def attention3d(q: Tensor, k: Tensor, impl: str = "auto", causal: bool = False, window: int = 0,
                deterministic: Optional[bool] = None) -> Tensor:
    return F_.cca3d_attention_forward(q, k, impl, deterministic, causal, window or None)


@attention3d.register_fake
def _(q, k, impl="auto", causal=False, window=0, deterministic=None):
    F_._time_window(causal, window or None)
    _format(impl, F_._attention_covered3d(q), q)
    B, _, T, H, W = q.shape
    return q.new_empty((B, T, H, W, H + W + T), dtype=torch.float32)


@torch.library.custom_op("cca::attention3d_backward", mutates_args=(), device_types="cuda")
def attention3d_backward(dattn: Tensor, attn: Tensor, q: Tensor, k: Tensor, impl: str = "auto", causal: bool = False,
                         window: int = 0, deterministic: Optional[bool] = None) -> Tuple[Tensor, Tensor]:
    return F_.cca3d_attention_backward(dattn, attn, q, k, impl, deterministic, causal, window or None)


@attention3d_backward.register_fake
def _(dattn, attn, q, k, impl="auto", causal=False, window=0, deterministic=None):
    fmt = _format(impl, F_._attention_covered3d(q), q)
    return torch.empty_like(q, memory_format=fmt), torch.empty_like(k, memory_format=fmt)


# ---- autograd.  Each backward op takes its forward op's arguments after the tensors (impl, causal, window, deterministic) in
#      the same order: they are saved as the forward got them and passed on, so the backward runs in the forward's mode.
def _values_setup(ctx, inputs, output):                 # forward, forward3d: (q, k, v, *mode) -> (out, lse)
    ctx.save_for_backward(*inputs[:3], *output)
    ctx.mode = inputs[3:]
    ctx.set_materialize_grads(False)                    # (lse passes no gradient: no zero tensor is filled for it)


def _map_setup(ctx, inputs, output):                    # attention, attention3d: (q, k, *mode) -> attn
    ctx.save_for_backward(output, *inputs[:2])
    ctx.mode = inputs[2:]


def _backward_by(op):
    def backward_(ctx, grad, *unused):                  # (the forward's lse passes no gradient)
        if grad is None:                                # only lse was used
            return (None,) * len(ctx.needs_input_grad)
        return (*op(grad, *ctx.saved_tensors, *ctx.mode),) + (None,) * len(ctx.mode)
    return backward_


forward.register_autograd(_backward_by(torch.ops.cca.backward), setup_context=_values_setup)
forward3d.register_autograd(_backward_by(torch.ops.cca.backward3d), setup_context=_values_setup)
attention.register_autograd(_backward_by(torch.ops.cca.attention_backward), setup_context=_map_setup)
attention3d.register_autograd(_backward_by(torch.ops.cca.attention3d_backward), setup_context=_map_setup)


# ---- the streaming step of the causal 3D op:  forward3d_step(q, k, v, k_cache, v_cache) -> (out[B,C,H,W], lse[B,H,W])
#      (channels-last out on the tensor-core path, contiguous on the generic kernel; no autograd: inference only).  The caches
#      are a ring: frames (-1: all N slots) past frames, frame j in slot (head + j) % N
@torch.library.custom_op("cca::forward3d_step", mutates_args=(), device_types="cuda")
def forward3d_step(q: Tensor, k: Tensor, v: Tensor, k_cache: Tensor, v_cache: Tensor, frames: int = -1,
                   head: int = 0) -> Tuple[Tensor, Tensor]:
    return F_.cca3d_step(q, k, v, k_cache, v_cache, frames=None if frames < 0 else frames, head=head)


@forward3d_step.register_fake
def _(q, k, v, k_cache, v_cache, frames=-1, head=0):
    S = k_cache.shape[2] if frames < 0 else frames
    return _out_lse(_format("auto", F_._covered3d(capi.CCA_WS_FORWARD, q, v, S + 1), q, v), q, v)
