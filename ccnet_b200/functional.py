"""Tensor-level entry points of the operator: ``cca_forward`` / ``cca_backward`` / ``cca``.

Host-side mirror of the reference's op boundary (cc_attention/functions.py:38-47): the caller
hands NCHW q, k, v; the extension returns out (and lse for backward).  Everything numerical
happens in the CUDA library behind the C ABI; PyTorch only owns memory, streams and autograd.
"""
from __future__ import annotations

import torch

from . import capi

_DTYPES = {torch.float32: capi.CCA_F32, torch.bfloat16: capi.CCA_BF16}
_IMPL_FLAGS = {"auto": capi.CCA_FLAG_AUTO, "simt": capi.CCA_FLAG_FORCE_SIMT, "tc": capi.CCA_FLAG_FORCE_TC}


def _check_inputs(q, k, v):
    if not (q.is_cuda and k.is_cuda and v.is_cuda):
        raise RuntimeError("ccnet_b200: criss-cross attention needs CUDA tensors on an H100 (sm_90) "
                           "(there is no CPU path in this package)")
    if q.dtype not in _DTYPES or k.dtype != q.dtype or v.dtype != q.dtype:
        raise RuntimeError(f"ccnet_b200: q,k,v must share dtype float32 or bfloat16, got "
                           f"{q.dtype},{k.dtype},{v.dtype}")
    if q.dim() != 4 or k.shape != q.shape or v.dim() != 4 or v.shape[0] != q.shape[0] or v.shape[2:] != q.shape[2:]:
        raise RuntimeError(f"ccnet_b200: expected q,k [B,Cq,H,W] and v [B,C,H,W], got "
                           f"{tuple(q.shape)},{tuple(k.shape)},{tuple(v.shape)}")
    if not (q.device == k.device == v.device):
        raise RuntimeError("ccnet_b200: q,k,v must be on the same device")


def _bf16_long_lines(dtype, H: int, W: int) -> bool:
    """bf16 I/O with lines longer than one 112-pixel tile: every output element of the tensor-core kernels is then the sum of
    up to 2*ceil(L/112) TMA reduce-adds, each rounded to bf16 in memory, in no fixed order -- measured at the 1e-2 budget
    (profiles/r02_parity_report.jsonl).  Such calls run on the fp32 kernels (bf16 values are exact in the bf16x3 split) and the
    result is rounded to bf16 ONCE.  CCA_B200_BF16_NATIVE=1 keeps the native bf16 kernels (the C ABI always does)."""
    import os
    return dtype == torch.bfloat16 and (H > 112 or W > 112) and not os.environ.get("CCA_B200_BF16_NATIVE")


def _stream_ptr(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def tc_eligible(B: int, Cq: int, C: int, H: int, W: int, dtype: torch.dtype) -> bool:
    """True if the wgmma (channels-last) kernels cover this problem, forward AND backward."""
    if dtype not in _DTYPES:
        return False
    lib = capi.load()
    return (lib.cca_b200_tc_supported(capi.CCA_WS_FORWARD, B, Cq, C, H, W, _DTYPES[dtype]) == 1
            and lib.cca_b200_tc_supported(capi.CCA_WS_BACKWARD, B, Cq, C, H, W, _DTYPES[dtype]) == 1)


def cca_forward(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, impl: str = "auto"):
    """One criss-cross step: returns (out[B,C,H,W], lse[B,H,W] fp32).

    ``impl``: "auto" (tensor-core kernels when they cover the shape, else the generic kernels),
    "tc" (tensor-core kernels or error), "simt" (generic kernels).  The tensor-core kernels work on
    channels-last memory (logical shape unchanged); inputs in another memory format are converted and
    the output is returned channels-last.  The generic kernels work on NCHW-contiguous memory.
    """
    _check_inputs(q, k, v)
    lib = capi.load()
    B, Cq, H, W = q.shape
    C = v.shape[1]
    dt = _DTYPES[q.dtype]
    flags = _IMPL_FLAGS[impl]
    use_tc = impl in ("auto", "tc") and lib.cca_b200_tc_supported(capi.CCA_WS_FORWARD, B, Cq, C, H, W, dt) == 1
    if impl == "tc" and not use_tc:
        raise RuntimeError(f"ccnet_b200: tensor-core kernels do not cover q{tuple(q.shape)} v{tuple(v.shape)} {q.dtype}")
    if use_tc and _bf16_long_lines(q.dtype, H, W):
        out32, lse = cca_forward(q.float(), k.float(), v.float(), impl)
        return out32.to(torch.bfloat16), lse
    if use_tc:
        fmt = torch.channels_last
        q, k, v = (t.contiguous(memory_format=fmt) for t in (q, k, v))
        flags |= capi.CCA_FLAG_NHWC
    else:
        fmt = torch.contiguous_format
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()   # reference calls .contiguous() too
    with torch.cuda.device(q.device):
        out = torch.empty_like(v, memory_format=fmt)
        lse = torch.empty((B, H, W), dtype=torch.float32, device=q.device)
        nws = lib.cca_b200_workspace_bytes(capi.CCA_WS_FORWARD, B, Cq, C, H, W, dt)
        ws = torch.empty((max(nws, 16),), dtype=torch.uint8, device=q.device)
        rc = lib.cca_b200_forward(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(),
                                  ws.data_ptr(), ws.numel(), B, Cq, C, H, W, dt, flags,
                                  _stream_ptr(q.device))
    capi.check(rc, "cca_b200_forward")
    return out, lse


def cca_backward(dout, q, k, v, out, lse, impl: str = "auto", want_delta: bool = False):
    """Gradients (dq, dk, dv) of ``cca_forward`` given dout and the saved forward tensors.
    ``want_delta``: also return delta[B,H,W] = <dout, out> per pixel as a 4th value when the tensor-core kernels ran (they
    leave it in the workspace; its sum is the gradient of the residual's gamma), else None.

    Same ``impl`` / memory-format rules as ``cca_forward``: the tensor-core kernels take and return
    channels-last tensors, the generic kernels NCHW-contiguous ones.
    """
    _check_inputs(q, k, v)
    lib = capi.load()
    if dout.dtype != q.dtype or out.dtype != q.dtype or dout.shape != v.shape or out.shape != v.shape:
        raise RuntimeError("ccnet_b200: dout/out must match v in shape and dtype")
    B, Cq, H, W = q.shape
    C = v.shape[1]
    dt = _DTYPES[q.dtype]
    flags = _IMPL_FLAGS[impl]
    if lse.dtype != torch.float32 or tuple(lse.shape) != (q.shape[0], q.shape[2], q.shape[3]) or lse.device != q.device:
        raise RuntimeError("ccnet_b200: lse must be the forward's float32 [B,H,W] tensor on the same device")
    if dout.device != q.device or out.device != q.device:
        raise RuntimeError("ccnet_b200: dout/out must be on the same device as q,k,v")
    use_tc = impl in ("auto", "tc") and lib.cca_b200_tc_supported(capi.CCA_WS_BACKWARD, B, Cq, C, H, W, dt) == 1
    if impl == "tc" and not use_tc:
        raise RuntimeError(f"ccnet_b200: tensor-core kernels do not cover q{tuple(q.shape)} v{tuple(v.shape)} {q.dtype}")
    if use_tc and _bf16_long_lines(q.dtype, H, W):
        res = cca_backward(dout.float(), q.float(), k.float(), v.float(), out.float(), lse, impl, want_delta)
        return tuple(g.to(torch.bfloat16) for g in res[:3]) + tuple(res[3:])
    if use_tc:
        fmt = torch.channels_last
        dout, q, k, v, out = (t.contiguous(memory_format=fmt) for t in (dout, q, k, v, out))
        flags |= capi.CCA_FLAG_NHWC
    else:
        fmt = torch.contiguous_format
        dout, q, k, v, out = (t.contiguous() for t in (dout, q, k, v, out))
    lse = lse.contiguous()
    with torch.cuda.device(q.device):
        dq = torch.empty_like(q, memory_format=fmt)
        dk = torch.empty_like(k, memory_format=fmt)
        dv = torch.empty_like(v, memory_format=fmt)
        nws = lib.cca_b200_workspace_bytes(capi.CCA_WS_BACKWARD, B, Cq, C, H, W, dt)
        ws = torch.empty((max(nws, 16),), dtype=torch.uint8, device=q.device)
        rc = lib.cca_b200_backward(dout.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(),
                                   lse.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(),
                                   ws.data_ptr(), ws.numel(), B, Cq, C, H, W, dt, flags,
                                   _stream_ptr(q.device))
    capi.check(rc, "cca_b200_backward")
    if want_delta:
        delta = ws[:B * H * W * 4].view(torch.float32).view(B, H, W) if use_tc else None
        return dq, dk, dv, delta
    return dq, dk, dv


def qkv_gemm_eligible(x: torch.Tensor, Cq: int) -> bool:
    """True if the hand-written wgmma projection GEMMs cover x [B,C,H,W] (fp32, C and Cq multiples of 64)."""
    return (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4
            and capi.load().cca_b200_qkv_supported(x.shape[1], Cq) == 1)


def _as_matrix_ptr(t: torch.Tensor) -> int:
    if not t.is_contiguous(memory_format=torch.channels_last) and not (t.dim() == 2 and t.is_contiguous()):
        raise RuntimeError("ccnet_b200: projection GEMMs need channels-last activations")
    return t.data_ptr()


def qkv_project(x, wq, bq, wk, bk, wv, bv):
    """q, k, v = the three 1x1 convs of cc_attention/functions.py:29,32,35 applied to channels-last x, as ONE wgmma GEMM
    launch emitting channels-last q, k, v.  fp32, C % 64 == 0, Cq % 64 == 0 (``qkv_gemm_eligible``)."""
    lib = capi.load()
    B, C, H, W = x.shape
    Cq = wq.shape[0]
    x = x.contiguous(memory_format=torch.channels_last)
    ws_w = [w.contiguous() for w in (wq, wk, wv)]
    bs = [b.contiguous() for b in (bq, bk, bv)]
    with torch.cuda.device(x.device):
        q = torch.empty((B, Cq, H, W), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        k = torch.empty_like(q, memory_format=torch.channels_last)
        v = torch.empty((B, C, H, W), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        nws = lib.cca_b200_qkv_workspace_bytes(C, Cq)
        ws = torch.empty((nws,), dtype=torch.uint8, device=x.device)
        rc = lib.cca_b200_qkv_project(_as_matrix_ptr(x), ws_w[0].data_ptr(), bs[0].data_ptr(), ws_w[1].data_ptr(), bs[1].data_ptr(),
                                      ws_w[2].data_ptr(), bs[2].data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr(),
                                      ws.data_ptr(), ws.numel(), B * H * W, C, Cq, _stream_ptr(x.device))
    capi.check(rc, "cca_b200_qkv_project")
    return q, k, v


def qkv_project_dgrad(dq, dk, dv, wq, wk, wv, scale=None):
    """dx = s (dq Wq + dk Wk + dv Wv) (input gradient of the three projections), channels-last fp32, one wgmma GEMM launch.
    ``scale``: optional one-element CUDA tensor s (the residual's gamma), folded into the packed weights."""
    lib = capi.load()
    B, C, H, W = dv.shape
    Cq = dq.shape[1]
    dq, dk, dv = (t.contiguous(memory_format=torch.channels_last) for t in (dq, dk, dv))
    ws_w = [w.contiguous() for w in (wq, wk, wv)]
    with torch.cuda.device(dv.device):
        dx = torch.empty_like(dv, memory_format=torch.channels_last)
        nws = lib.cca_b200_qkv_workspace_bytes(C, Cq)
        ws = torch.empty((nws,), dtype=torch.uint8, device=dv.device)
        rc = lib.cca_b200_qkv_project_dgrad(dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), ws_w[0].data_ptr(), ws_w[1].data_ptr(),
                                            ws_w[2].data_ptr(), scale.data_ptr() if scale is not None else None, dx.data_ptr(),
                                            ws.data_ptr(), ws.numel(), B * H * W, C, Cq, 0, _stream_ptr(dv.device))
    capi.check(rc, "cca_b200_qkv_project_dgrad")
    return dx


def qkv_wgrad_eligible(C: int, Cq: int) -> bool:
    return capi.load().cca_b200_qkv_wgrad_supported(C, Cq) == 1


def qkv_project_wgrad(x, dq, dk, dv, scale=None):
    """(dWq, dbq, dWk, dbk, dWv, dbv) = s * (gradients of the three 1x1 convs' parameters), one split-K wgmma launch."""
    lib = capi.load()
    B, C, H, W = x.shape
    Cq = dq.shape[1]
    x, dq, dk, dv = (t.contiguous(memory_format=torch.channels_last) for t in (x, dq, dk, dv))
    with torch.cuda.device(x.device):
        dwq = torch.empty((Cq, C), dtype=x.dtype, device=x.device)
        dwk = torch.empty((Cq, C), dtype=x.dtype, device=x.device)
        dwv = torch.empty((C, C), dtype=x.dtype, device=x.device)
        db = torch.empty((2 * Cq + C,), dtype=x.dtype, device=x.device)
        rc = lib.cca_b200_qkv_project_wgrad(x.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(),
                                            scale.data_ptr() if scale is not None else None, dwq.data_ptr(), dwk.data_ptr(),
                                            dwv.data_ptr(), db.data_ptr(), B * H * W, C, Cq, _stream_ptr(x.device))
    capi.check(rc, "cca_b200_qkv_project_wgrad")
    return dwq, db[:Cq], dwk, db[Cq:2 * Cq], dwv, db[2 * Cq:]


class _CCAFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, impl):
        out, lse = cca_forward(q, k, v, impl)
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.impl = impl
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, out, lse = ctx.saved_tensors
        dq, dk, dv = cca_backward(dout, q, k, v, out, lse, ctx.impl)
        return dq, dk, dv, None


def cca(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, impl: str = "auto") -> torch.Tensor:
    """Differentiable criss-cross attention step (out only)."""
    return _CCAFunction.apply(q, k, v, impl)
