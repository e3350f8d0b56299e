"""Tensor-level entry points of the operator: ``cca_forward`` / ``cca_backward`` / ``cca``.

Host-side mirror of the reference's op boundary (cc_attention/functions.py:38-47): the caller
hands NCHW q, k, v; the extension returns out (and lse for backward).  Everything numerical
happens in the CUDA library behind the C ABI; PyTorch only owns memory, streams and autograd.
"""
from __future__ import annotations

import os

import torch

from . import capi

_DTYPES = {torch.float32: capi.CCA_F32, torch.bfloat16: capi.CCA_BF16, torch.float16: capi.CCA_F16}
_IMPL_FLAGS = {"auto": capi.CCA_FLAG_AUTO, "simt": capi.CCA_FLAG_FORCE_SIMT, "tc": capi.CCA_FLAG_FORCE_TC}

#: Bytes of partial-plane workspace one deterministic call may allocate (lines longer than 112 pixels).  A batch that would
#: need more runs in groups of samples; a sample's result does not depend on the batch it is in, so the bits are the same.
deterministic_workspace_cap = 1 << 30


def _resolve_deterministic(deterministic) -> bool:
    """``deterministic=None`` follows ``torch.use_deterministic_algorithms``."""
    return torch.are_deterministic_algorithms_enabled() if deterministic is None else bool(deterministic)


def _workspace(nbytes: int, device) -> torch.Tensor:
    """Device scratch of the C ABI calls.  The kernels write every byte they read, so torch's deterministic mode need not fill
    it first (its ``torch.empty`` fill would otherwise touch up to ``deterministic_workspace_cap`` bytes per call).  The fill
    switch is process-wide: a ``torch.empty`` another thread runs meanwhile may come back unfilled."""
    if not torch.are_deterministic_algorithms_enabled():
        return torch.empty((max(nbytes, 16),), dtype=torch.uint8, device=device)
    import torch.utils.deterministic as td
    fill = td.fill_uninitialized_memory
    td.fill_uninitialized_memory = False
    try:
        return torch.empty((max(nbytes, 16),), dtype=torch.uint8, device=device)
    finally:
        td.fill_uninitialized_memory = fill


def _check_inputs(q, k, v=None, rank: int = 4):
    """q, k [B,Cq,H,W] (rank 5: [B,Cq,T,H,W]) and, when given, v [B,C,...]: CUDA tensors of one dtype on one device"""
    ts = (q, k) if v is None else (q, k, v)
    names = ",".join("qkv"[:len(ts)])
    if not all(t.is_cuda for t in ts):
        raise RuntimeError("ccnet_b200: criss-cross attention needs CUDA tensors on an H100 (sm_90) "
                           "(there is no CPU path in this package)")
    if q.dtype not in _DTYPES or any(t.dtype != q.dtype for t in ts):
        raise RuntimeError(f"ccnet_b200: {names} must share dtype float32, bfloat16 or float16, got "
                           + ",".join(str(t.dtype) for t in ts))
    if q.dim() != rank or k.shape != q.shape or (v is not None and (v.dim() != rank or v.shape[0] != q.shape[0]
                                                                    or v.shape[2:] != q.shape[2:])):
        s = "T,H,W" if rank == 5 else "H,W"
        raise RuntimeError(f"ccnet_b200: expected q,k [B,Cq,{s}]" + ("" if v is None else f" and v [B,C,{s}]") + ", got "
                           + ",".join(str(tuple(t.shape)) for t in ts))
    if any(t.device != q.device for t in ts):
        raise RuntimeError(f"ccnet_b200: {names} must be on the same device")


def _check_saved(q, v, dout, out, lse):
    """a backward's dout and the forward's out (both like v) and lse (float32 [B,H,W], or [B,T,H,W])"""
    if dout.dtype != q.dtype or out.dtype != q.dtype or dout.shape != v.shape or out.shape != v.shape:
        raise RuntimeError("ccnet_b200: dout/out must match v in shape and dtype")
    if dout.device != q.device or out.device != q.device:
        raise RuntimeError("ccnet_b200: dout/out must be on the same device as q,k,v")
    if lse.dtype != torch.float32 or tuple(lse.shape) != (q.shape[0], *q.shape[2:]) or lse.device != q.device:
        s = "T,H,W" if q.dim() == 5 else "H,W"
        raise RuntimeError(f"ccnet_b200: lse must be the forward's float32 [B,{s}] tensor on the same device")


def _plan(impl: str, det: bool, covered, q, v=None, causal: bool = False):
    """(use_tc, flags, memory format) of a call: the tensor-core kernels on channels-last memory where ``covered()``, the
    op's coverage query, says they take the shape and ``impl`` allows them, else the generic kernels on contiguous memory.
    impl="tc" on a shape the tensor-core kernels do not cover raises.  ``causal`` adds CCA_FLAG_CAUSAL (3D ops).  The real
    calls and the fake implementations of ``ccnet_b200.ops`` both take their memory format from here."""
    use_tc = impl in ("auto", "tc") and covered()
    if impl == "tc" and not use_tc:
        shapes = f"q{tuple(q.shape)}" + ("" if v is None else f" v{tuple(v.shape)}")
        raise RuntimeError(f"ccnet_b200: tensor-core kernels do not cover {shapes} {q.dtype}")
    flags = (_IMPL_FLAGS[impl] | (capi.CCA_FLAG_NHWC if use_tc else 0) | (capi.CCA_FLAG_DETERMINISTIC if det else 0)
             | (capi.CCA_FLAG_CAUSAL if causal else 0))
    fmt = (torch.channels_last_3d if q.dim() == 5 else torch.channels_last) if use_tc else torch.contiguous_format
    return use_tc, flags, fmt


# The coverage queries of the ops for ``_plan``, evaluated only when ``impl`` allows the tensor-core kernels.
def _covered(which, q, v):
    """the 2D op (``which``: CCA_WS_FORWARD or CCA_WS_BACKWARD) on q [B,Cq,H,W], v [B,C,H,W]"""
    B, Cq, H, W = q.shape
    return lambda: (q.dtype in _DTYPES
                    and capi.load().cca_b200_tc_supported(which, B, Cq, v.shape[1], H, W, _DTYPES[q.dtype]) == 1)


def _attention_covered(q):
    """the 2D map on q [B,Cq,H,W]"""
    return lambda: attention_tc_eligible(*q.shape, q.dtype)


def _covered3d(which, q, v, T: int):
    """the 3D op on a clip of T frames: q [B,Cq,T,H,W], or the new frame [B,Cq,H,W] of a step with T = S + 1"""
    B, Cq, H, W = q.shape[0], q.shape[1], q.shape[-2], q.shape[-1]
    return lambda: (q.dtype in _DTYPES
                    and capi.load().cca_b200_tc3d_supported(which, B, Cq, v.shape[1], T, H, W, _DTYPES[q.dtype]) == 1)


def _attention_covered3d(q):
    """the 3D map on q [B,Cq,T,H,W]"""
    return lambda: attention3d_tc_eligible(*q.shape, q.dtype)


def _time_window(causal: bool, window) -> int:
    """The C ABI's window argument of a 3D call: 0 for ``window=None`` (every past frame), else W >= 1, causal mode only."""
    if window is None:
        return 0
    if not causal:
        raise ValueError("ccnet_b200: a time window needs causal=True (windows of the bidirectional op are not supported)")
    if isinstance(window, bool) or int(window) != window or window < 1:
        raise ValueError(f"ccnet_b200: window must be an integer >= 1 or None, got {window!r}")
    return int(window)


def _ws3d(which, B, Cq, C, T, H, W, window, dt, flags) -> int:
    """cca_b200_workspace_bytes3d for the dimensions of a *_window call (the window does not change it)"""
    return capi.load().cca_b200_workspace_bytes3d(which, B, Cq, C, T, H, W, dt, flags)


def _attn_ws3d(backward, B, Cq, T, H, W, window, dt, flags) -> int:
    """cca_b200_attention_workspace_bytes3d for the dimensions of a *_window call"""
    return capi.load().cca_b200_attention_workspace_bytes3d(backward, B, Cq, T, H, W, dt, flags)


def _upcast(dtype, H: int, W: int, deterministic: bool, T: int = 1) -> bool:
    """16-bit calls of the tensor-core path that run on the fp32 kernels on upcast tensors (bf16 and fp16 values are exact in
    the bf16x3 split), the result rounded to the 16-bit type ONCE:
    - lines longer than one 112-pixel tile: every output element of the native kernels is the sum of up to 2*ceil(L/112) TMA
      reduce-adds, each rounded to the 16-bit type in memory, in no fixed order -- at the 1e-2 budget for bf16.
    - bf16 with T > 1 (the 3D op and its attention map's backward): the time pass adds onto out, dq, dk and dv after the
      2D passes have rounded them to the I/O type, a third rounding of every output element; in bf16 that puts the
      emulated floor at up to 0.73 of the 1e-2 budget (tests/test_cca3d_host.py), in fp16 at a third of its budget (the
      map's dq, dk: tests/test_attention3d_host.py).  At T = 1 the time pass adds nothing and the native kernels give the
      2D op's bits.
    CCA_B200_BF16_NATIVE=1 keeps the native bf16 and fp16 kernels (the C ABI always does), except in deterministic mode on
    long lines: only the fp32 kernels have it there."""
    if dtype not in (torch.bfloat16, torch.float16):
        return False
    native = bool(os.environ.get("CCA_B200_BF16_NATIVE"))
    if H > 112 or W > 112:
        return deterministic or not native
    return dtype == torch.bfloat16 and T > 1 and not native


def _grouped_call(fn, ws_query, which, tensors, dims, dt, flags, each=None):
    """``fn(*pointers of the tensors, workspace, its bytes, n, *dims, dt, flags, stream)``, a C ABI entry point, over batch
    slices [b0, b1) of the tensors, each with a workspace of ``ws_query(which, n, *dims, dt, flags)`` bytes.  One slice
    unless the call is deterministic and needs partial planes: then the planes of a slice, per sample the workspace with the
    flag minus the one without it, stay under ``deterministic_workspace_cap``.  ``each(b0, b1, ws)`` runs after each
    slice's call."""
    B, device = tensors[0].shape[0], tensors[0].device
    groups = [(0, B)]
    if flags & capi.CCA_FLAG_DETERMINISTIC:
        per_sample = (ws_query(which, 1, *dims, dt, flags)
                      - ws_query(which, 1, *dims, dt, flags & ~capi.CCA_FLAG_DETERMINISTIC))
        if per_sample > 0:
            g = max(1, deterministic_workspace_cap // per_sample)
            groups = [(b0, min(B, b0 + g)) for b0 in range(0, B, g)]
    stream = _stream_ptr(device)
    for b0, b1 in groups:
        ws = _workspace(ws_query(which, b1 - b0, *dims, dt, flags), device)
        rc = fn(*(t[b0:b1].data_ptr() for t in tensors), ws.data_ptr(), ws.numel(), b1 - b0, *dims, dt, flags, stream)
        capi.check(rc, fn.__name__)
        if each is not None:
            each(b0, b1, ws)


def _stream_ptr(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def tc_eligible(B: int, Cq: int, C: int, H: int, W: int, dtype: torch.dtype) -> bool:
    """True if the wgmma (channels-last) kernels cover this problem, forward AND backward."""
    if dtype not in _DTYPES:
        return False
    lib = capi.load()
    return (lib.cca_b200_tc_supported(capi.CCA_WS_FORWARD, B, Cq, C, H, W, _DTYPES[dtype]) == 1
            and lib.cca_b200_tc_supported(capi.CCA_WS_BACKWARD, B, Cq, C, H, W, _DTYPES[dtype]) == 1)


def cca_forward(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, impl: str = "auto", deterministic=None):
    """One criss-cross step: returns (out[B,C,H,W], lse[B,H,W] fp32).

    ``impl``: "auto" (tensor-core kernels when they cover the shape, else the generic kernels),
    "tc" (tensor-core kernels or error), "simt" (generic kernels).  The tensor-core kernels work on
    channels-last memory (logical shape unchanged); inputs in another memory format are converted and
    the output is returned channels-last.  The generic kernels work on NCHW-contiguous memory.

    ``deterministic``: bit-reproducible results (CCA_FLAG_DETERMINISTIC); None follows
    ``torch.are_deterministic_algorithms_enabled()``.
    """
    _check_inputs(q, k, v)
    det = _resolve_deterministic(deterministic)
    lib = capi.load()
    B, Cq, H, W = q.shape
    C = v.shape[1]
    dt = _DTYPES[q.dtype]
    use_tc, flags, fmt = _plan(impl, det, _covered(capi.CCA_WS_FORWARD, q, v), q, v)
    if use_tc and _upcast(q.dtype, H, W, det):
        out32, lse = cca_forward(q.float(), k.float(), v.float(), impl, det)
        return out32.to(q.dtype), lse
    q, k, v = (t.contiguous(memory_format=fmt) for t in (q, k, v))     # (the reference calls .contiguous() too)
    with torch.cuda.device(q.device):
        out = torch.empty_like(v, memory_format=fmt)
        lse = torch.empty((B, H, W), dtype=torch.float32, device=q.device)
        _grouped_call(lib.cca_b200_forward, lib.cca_b200_workspace_bytes_ex, capi.CCA_WS_FORWARD, (q, k, v, out, lse),
                      (Cq, C, H, W), dt, flags)
    return out, lse


def cca_backward(dout, q, k, v, out, lse, impl: str = "auto", want_delta: bool = False, deterministic=None):
    """Gradients (dq, dk, dv) of ``cca_forward`` given dout and the saved forward tensors.
    ``want_delta``: also return delta[B,H,W] = <dout, out> per pixel as a 4th value when the tensor-core kernels ran (they
    leave it in the workspace; its sum is the gradient of the residual's gamma), else None.

    Same ``impl`` / memory-format / ``deterministic`` rules as ``cca_forward``: the tensor-core kernels take and return
    channels-last tensors, the generic kernels NCHW-contiguous ones.
    """
    _check_inputs(q, k, v)
    _check_saved(q, v, dout, out, lse)
    det = _resolve_deterministic(deterministic)
    lib = capi.load()
    B, Cq, H, W = q.shape
    C = v.shape[1]
    dt = _DTYPES[q.dtype]
    use_tc, flags, fmt = _plan(impl, det, _covered(capi.CCA_WS_BACKWARD, q, v), q, v)
    if use_tc and _upcast(q.dtype, H, W, det):
        res = cca_backward(dout.float(), q.float(), k.float(), v.float(), out.float(), lse, impl, want_delta, det)
        return tuple(g.to(q.dtype) for g in res[:3]) + tuple(res[3:])
    dout, q, k, v, out = (t.contiguous(memory_format=fmt) for t in (dout, q, k, v, out))
    lse = lse.contiguous()
    delta = None

    def keep_delta(b0, b1, ws):             # (the delta of each slice is at the start of its workspace)
        nonlocal delta
        part = ws[:(b1 - b0) * H * W * 4].view(torch.float32).view(b1 - b0, H, W)
        if b1 - b0 == B:
            delta = part
            return
        if delta is None:
            delta = torch.empty((B, H, W), dtype=torch.float32, device=q.device)
        delta[b0:b1].copy_(part)

    with torch.cuda.device(q.device):
        dq = torch.empty_like(q, memory_format=fmt)
        dk = torch.empty_like(k, memory_format=fmt)
        dv = torch.empty_like(v, memory_format=fmt)
        _grouped_call(lib.cca_b200_backward, lib.cca_b200_workspace_bytes_ex, capi.CCA_WS_BACKWARD,
                      (dout, q, k, v, out, lse, dq, dk, dv), (Cq, C, H, W), dt, flags, keep_delta if want_delta and use_tc else None)
    return (dq, dk, dv, delta) if want_delta else (dq, dk, dv)


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


def qkv_project_wgrad(x, dq, dk, dv, scale=None, deterministic=None):
    """(dWq, dbq, dWk, dbk, dWv, dbv) = s * (gradients of the three 1x1 convs' parameters), one split-K wgmma launch.
    ``deterministic`` (None: ``torch.are_deterministic_algorithms_enabled()``): the splits' partials are added in a fixed
    order (reproducible on one GPU model) instead of with atomics."""
    lib = capi.load()
    det = _resolve_deterministic(deterministic)
    B, C, H, W = x.shape
    Cq = dq.shape[1]
    x, dq, dk, dv = (t.contiguous(memory_format=torch.channels_last) for t in (x, dq, dk, dv))
    with torch.cuda.device(x.device):
        dwq = torch.empty((Cq, C), dtype=x.dtype, device=x.device)
        dwk = torch.empty((Cq, C), dtype=x.dtype, device=x.device)
        dwv = torch.empty((C, C), dtype=x.dtype, device=x.device)
        db = torch.empty((2 * Cq + C,), dtype=x.dtype, device=x.device)
        nws = lib.cca_b200_qkv_wgrad_workspace_bytes(C, Cq) if det else 0
        ws = _workspace(nws, x.device) if det else None
        rc = lib.cca_b200_qkv_project_wgrad_ex(x.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(),
                                               scale.data_ptr() if scale is not None else None, dwq.data_ptr(),
                                               dwk.data_ptr(), dwv.data_ptr(), db.data_ptr(), B * H * W, C, Cq,
                                               ws.data_ptr() if det else None, nws,
                                               capi.CCA_FLAG_DETERMINISTIC if det else 0, _stream_ptr(x.device))
    capi.check(rc, "cca_b200_qkv_project_wgrad_ex")
    return dwq, db[:Cq], dwk, db[Cq:2 * Cq], dwv, db[2 * Cq:]


def cca(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, impl: str = "auto", deterministic=None) -> torch.Tensor:
    """Differentiable criss-cross attention step (out only).  ``deterministic``: as for ``cca_forward``; the mode is fixed
    when the forward runs and the backward uses it too."""
    _check_inputs(q, k, v)
    return torch.ops.cca.forward(q, k, v, impl, _resolve_deterministic(deterministic))[0]


# ---------------------------------------------------------------------------------------------------------------------
# attention map (cc_attention/functions.py:40, the softmax output `concate`) and its gradient
# ---------------------------------------------------------------------------------------------------------------------
def attention_tc_eligible(B: int, Cq: int, H: int, W: int, dtype: torch.dtype) -> bool:
    """True if the wgmma (channels-last) attention-map kernels cover this problem."""
    return dtype in _DTYPES and capi.load().cca_b200_attention_tc_supported(B, Cq, H, W, _DTYPES[dtype]) == 1


def cca_attention_forward(q: torch.Tensor, k: torch.Tensor, impl: str = "auto", deterministic=None) -> torch.Tensor:
    """The attention map of one criss-cross step, attn[B,H,W,H+W] float32 (the reference's ``concate``): attn[b,h,w,g] is
    the weight of column key (g, w) for g < H (0 at g == h) and of row key (h, g - H) for g >= H.

    ``impl`` as for ``cca_forward``.  Every map element is written once, so the result is the same in every mode;
    ``deterministic`` only sets the flag the C ABI is called with."""
    _check_inputs(q, k)
    det = _resolve_deterministic(deterministic)
    lib = capi.load()
    B, Cq, H, W = q.shape
    dt = _DTYPES[q.dtype]
    use_tc, flags, fmt = _plan(impl, det, _attention_covered(q), q)
    q, k = (t.contiguous(memory_format=fmt) for t in (q, k))
    with torch.cuda.device(q.device):
        attn = torch.empty((B, H, W, H + W), dtype=torch.float32, device=q.device)
        ws = _workspace(lib.cca_b200_attention_workspace_bytes(0, B, Cq, H, W, dt, flags), q.device)
        rc = lib.cca_b200_attention_forward(q.data_ptr(), k.data_ptr(), attn.data_ptr(), ws.data_ptr(), ws.numel(),
                                            B, Cq, H, W, dt, flags, _stream_ptr(q.device))
        capi.check(rc, "cca_b200_attention_forward")
    return attn


def cca_attention_backward(dattn, attn, q, k, impl: str = "auto", deterministic=None):
    """Gradients (dq, dk) of ``cca_attention_forward`` given dattn = dL/dattn and the forward's map:
    dS = attn * (dattn - rho), rho = sum_j attn dattn;  dq = dS k,  dk = dS^T q.  Same ``impl`` / memory-format /
    ``deterministic`` rules as ``cca_backward``."""
    _check_inputs(q, k)
    det = _resolve_deterministic(deterministic)
    lib = capi.load()
    B, Cq, H, W = q.shape
    for name, t in (("attn", attn), ("dattn", dattn)):
        if t.dtype != torch.float32 or tuple(t.shape) != (B, H, W, H + W) or t.device != q.device:
            raise RuntimeError(f"ccnet_b200: {name} must be a float32 [B,H,W,H+W] tensor on the device of q, k")
    dt = _DTYPES[q.dtype]
    use_tc, flags, fmt = _plan(impl, det, _attention_covered(q), q)
    if use_tc and _upcast(q.dtype, H, W, det):
        dq, dk = cca_attention_backward(dattn, attn, q.float(), k.float(), impl, det)
        return dq.to(q.dtype), dk.to(q.dtype)
    q, k = (t.contiguous(memory_format=fmt) for t in (q, k))
    dattn, attn = dattn.contiguous(), attn.contiguous()
    with torch.cuda.device(q.device):
        dq = torch.empty_like(q, memory_format=fmt)
        dk = torch.empty_like(k, memory_format=fmt)
        _grouped_call(lib.cca_b200_attention_backward, lib.cca_b200_attention_workspace_bytes, 1, (dattn, attn, q, k, dq, dk),
                      (Cq, H, W), dt, flags)
    return dq, dk


def cca_attention(q: torch.Tensor, k: torch.Tensor, impl: str = "auto", deterministic=None) -> torch.Tensor:
    """Differentiable attention map attn[B,H,W,H+W] (float32) of one criss-cross step; the gradient flows to q and k.
    ``deterministic``: as for ``cca``; the mode is fixed when the forward runs and the backward uses it too."""
    _check_inputs(q, k)
    return torch.ops.cca.attention(q, k, impl, _resolve_deterministic(deterministic))


# ---------------------------------------------------------------------------------------------------------------------
# criss-cross attention over clips (the 3D op): column, row and time branches under one softmax
# ---------------------------------------------------------------------------------------------------------------------
def tc3d_eligible(B: int, Cq: int, C: int, T: int, H: int, W: int, dtype: torch.dtype) -> bool:
    """True if the 3D op's kernels cover this problem (the 2D tensor-core shapes for B*T frames, 1 <= T <= 32)."""
    return dtype in _DTYPES and capi.load().cca_b200_tc3d_supported(capi.CCA_WS_FORWARD, B, Cq, C, T, H, W, _DTYPES[dtype]) == 1


def cca3d_forward(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, impl: str = "auto", deterministic=None,
                  causal: bool = False, window=None):
    """Criss-cross attention over clips: returns (out[B,C,T,H,W], lse[B,T,H,W] fp32).  q, k are [B,Cq,T,H,W], v [B,C,T,H,W].
    Pixel (b,t,h,w) attends to its column (self masked), its row and its time line (self masked), one softmax over the
    H + W + T logits.  At T = 1 this is ``cca_forward`` on every frame.

    ``impl``: "auto" (the tensor-core path where ``tc3d_eligible``, else the generic kernels), "tc" (tensor-core path or
    error), "simt" (generic kernels: any Cq and C, H + W + T - 2 <= 2048).  The tensor-core path works on channels_last_3d
    memory (inputs in another format are converted, the output is channels_last_3d), the generic kernels on contiguous
    NCDHW memory.  ``deterministic`` as for ``cca_forward``.

    ``causal``: the time keys of frame t are the frames s < t only (CCA_FLAG_CAUSAL); frame 0 then has no time key and is
    ``cca_forward`` on its frame.  For streaming inference, ``cca3d_step`` produces one new frame from cached keys and values.

    ``window`` (causal mode only; None: every past frame): W >= 1 limits the time keys of frame t to the frames
    t - W <= s < t.  With W >= T - 1 the result is bit for bit that of ``window=None``.  The generic kernels then take
    H + W_img - 1 + min(W, T - 1) <= 2048, so a windowed clip may have any length; ``cca3d_step`` on a ring of the last W
    frames streams the same op."""
    _check_inputs(q, k, v, rank=5)
    win = _time_window(causal, window)
    det = _resolve_deterministic(deterministic)
    lib = capi.load()
    B, Cq, T, H, W = q.shape
    C = v.shape[1]
    dt = _DTYPES[q.dtype]
    use_tc, flags, fmt = _plan(impl, det, _covered3d(capi.CCA_WS_FORWARD, q, v, T), q, v, causal)
    if use_tc and _upcast(q.dtype, H, W, det, T):
        out32, lse = cca3d_forward(q.float(), k.float(), v.float(), impl, det, causal, window)
        return out32.to(q.dtype), lse
    q, k, v = (t.contiguous(memory_format=fmt) for t in (q, k, v))
    with torch.cuda.device(q.device):
        out = torch.empty_like(v, memory_format=fmt)
        lse = torch.empty((B, T, H, W), dtype=torch.float32, device=q.device)
        _grouped_call(lib.cca_b200_forward3d_window, _ws3d, capi.CCA_WS_FORWARD, (q, k, v, out, lse), (Cq, C, T, H, W, win), dt,
                      flags)
    return out, lse


def cca3d_backward(dout, q, k, v, out, lse, impl: str = "auto", deterministic=None, causal: bool = False, window=None):
    """Gradients (dq, dk, dv) of ``cca3d_forward`` given dout and the saved forward tensors.  Same ``impl`` / memory-format /
    ``deterministic`` / ``causal`` / ``window`` rules as ``cca3d_forward``."""
    _check_inputs(q, k, v, rank=5)
    _check_saved(q, v, dout, out, lse)
    win = _time_window(causal, window)
    det = _resolve_deterministic(deterministic)
    lib = capi.load()
    B, Cq, T, H, W = q.shape
    C = v.shape[1]
    dt = _DTYPES[q.dtype]
    use_tc, flags, fmt = _plan(impl, det, _covered3d(capi.CCA_WS_BACKWARD, q, v, T), q, v, causal)
    if use_tc and _upcast(q.dtype, H, W, det, T):
        res = cca3d_backward(dout.float(), q.float(), k.float(), v.float(), out.float(), lse, impl, det, causal, window)
        return tuple(g.to(q.dtype) for g in res)
    dout, q, k, v, out = (t.contiguous(memory_format=fmt) for t in (dout, q, k, v, out))
    lse = lse.contiguous()
    with torch.cuda.device(q.device):
        dq = torch.empty_like(q, memory_format=fmt)
        dk = torch.empty_like(k, memory_format=fmt)
        dv = torch.empty_like(v, memory_format=fmt)
        _grouped_call(lib.cca_b200_backward3d_window, _ws3d, capi.CCA_WS_BACKWARD, (dout, q, k, v, out, lse, dq, dk, dv),
                      (Cq, C, T, H, W, win), dt, flags)
    return dq, dk, dv


def cca3d(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, impl: str = "auto", deterministic=None,
          causal: bool = False, window=None) -> torch.Tensor:
    """Differentiable criss-cross attention over clips (out only); see ``cca3d_forward``.  The ``causal`` mode and
    ``window`` of the forward are kept for the backward."""
    _check_inputs(q, k, v, rank=5)
    win = _time_window(causal, window)
    return torch.ops.cca.forward3d(q, k, v, bool(causal), win, impl, _resolve_deterministic(deterministic))[0]


# ---------------------------------------------------------------------------------------------------------------------
# attention map of criss-cross attention over clips and its gradient
# ---------------------------------------------------------------------------------------------------------------------
def attention3d_tc_eligible(B: int, Cq: int, T: int, H: int, W: int, dtype: torch.dtype) -> bool:
    """True if the tensor-core (channels_last_3d) kernels of the 3D attention map cover this problem."""
    return dtype in _DTYPES and capi.load().cca_b200_attention_tc3d_supported(B, Cq, T, H, W, _DTYPES[dtype]) == 1


def cca3d_attention_forward(q: torch.Tensor, k: torch.Tensor, impl: str = "auto", deterministic=None,
                            causal: bool = False, window=None) -> torch.Tensor:
    """The attention map of ``cca3d_forward``, attn[B,T,H,W,H+W+T] float32: attn[b,t,h,w,g] is the weight of column key
    (t, g, w) for g < H (0 at g == h), of row key (t, h, g - H) for H <= g < H + W and of time key (g - H - W, h, w) after
    that (0 at g - H - W == t).  It is normalised by the lse of ``cca3d_forward``; at T = 1, attn[..., :H+W] is
    ``cca_attention_forward`` of every frame and attn[..., H+W] is 0.

    ``impl`` as for ``cca3d_forward`` (the generic kernels take any Cq and shape).  Every map element is written once, so
    the result is the same in every mode; ``deterministic`` only sets the flag the C ABI is called with.  ``causal``: the map
    of ``cca3d_forward(..., causal=True)``, same layout, time entries H + W + s with s >= t exactly 0.  ``window``: that of
    ``cca3d_forward(..., causal=True, window=W)``; time entries outside [t - W, t) are exactly 0."""
    _check_inputs(q, k, rank=5)
    win = _time_window(causal, window)
    det = _resolve_deterministic(deterministic)
    lib = capi.load()
    B, Cq, T, H, W = q.shape
    dt = _DTYPES[q.dtype]
    use_tc, flags, fmt = _plan(impl, det, _attention_covered3d(q), q, causal=causal)
    q, k = (t.contiguous(memory_format=fmt) for t in (q, k))
    with torch.cuda.device(q.device):
        attn = torch.empty((B, T, H, W, H + W + T), dtype=torch.float32, device=q.device)
        ws = _workspace(lib.cca_b200_attention_workspace_bytes3d(0, B, Cq, T, H, W, dt, flags), q.device)
        rc = lib.cca_b200_attention_forward3d_window(q.data_ptr(), k.data_ptr(), attn.data_ptr(), ws.data_ptr(), ws.numel(),
                                                     B, Cq, T, H, W, win, dt, flags, _stream_ptr(q.device))
        capi.check(rc, "cca_b200_attention_forward3d_window")
    return attn


def cca3d_attention_backward(dattn, attn, q, k, impl: str = "auto", deterministic=None, causal: bool = False, window=None):
    """Gradients (dq, dk) of ``cca3d_attention_forward`` given dattn = dL/dattn and the forward's map, in the closed form
    of ``cca_attention_backward`` over the H + W + T entries of a row.  Same ``impl`` / memory-format / ``deterministic`` /
    ``causal`` / ``window`` rules as ``cca3d_backward``."""
    _check_inputs(q, k, rank=5)
    win = _time_window(causal, window)
    det = _resolve_deterministic(deterministic)
    lib = capi.load()
    B, Cq, T, H, W = q.shape
    for name, t in (("attn", attn), ("dattn", dattn)):
        if t.dtype != torch.float32 or tuple(t.shape) != (B, T, H, W, H + W + T) or t.device != q.device:
            raise RuntimeError(f"ccnet_b200: {name} must be a float32 [B,T,H,W,H+W+T] tensor on the device of q, k")
    dt = _DTYPES[q.dtype]
    use_tc, flags, fmt = _plan(impl, det, _attention_covered3d(q), q, causal=causal)
    if use_tc and _upcast(q.dtype, H, W, det, T):
        dq, dk = cca3d_attention_backward(dattn, attn, q.float(), k.float(), impl, det, causal, window)
        return dq.to(q.dtype), dk.to(q.dtype)
    q, k = (t.contiguous(memory_format=fmt) for t in (q, k))
    dattn, attn = dattn.contiguous(), attn.contiguous()
    with torch.cuda.device(q.device):
        dq = torch.empty_like(q, memory_format=fmt)
        dk = torch.empty_like(k, memory_format=fmt)
        _grouped_call(lib.cca_b200_attention_backward3d_window, _attn_ws3d, 1, (dattn, attn, q, k, dq, dk), (Cq, T, H, W, win), dt,
                      flags)
    return dq, dk


def cca3d_attention(q: torch.Tensor, k: torch.Tensor, impl: str = "auto", deterministic=None,
                    causal: bool = False, window=None) -> torch.Tensor:
    """Differentiable attention map attn[B,T,H,W,H+W+T] (float32) of criss-cross attention over clips; the gradient flows
    to q and k.  ``deterministic``, ``causal`` and ``window``: as for ``cca3d``; they are fixed when the forward runs and
    the backward uses them too."""
    _check_inputs(q, k, rank=5)
    win = _time_window(causal, window)
    return torch.ops.cca.attention3d(q, k, impl, bool(causal), win, _resolve_deterministic(deterministic))


# ---------------------------------------------------------------------------------------------------------------------
# streaming step of causal criss-cross attention over clips
# ---------------------------------------------------------------------------------------------------------------------
def cca3d_step(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor,
               impl: str = "auto", deterministic=None, frames=None, head: int = 0):
    """One new frame of causal criss-cross attention over clips, for streaming inference: returns (out[B,C,H,W],
    lse[B,H,W] fp32).  q, k [B,Cq,H,W] and v [B,C,H,W] are the new frame's; k_cache [B,Cq,S,H,W] and v_cache [B,C,S,H,W]
    the keys and values of the S previous frames in time order.  By definition the result is frame S of
    ``cca3d_forward(..., causal=True)`` on the clip whose frames 0..S-1 have those keys and values and whose frame S has
    k, v (the past frames' queries do not enter); S = 0 is ``cca_forward`` on the frame.

    ``impl`` / ``deterministic`` as for ``cca3d_forward``: the tensor-core path (channels-last frame, channels_last_3d
    caches, S <= 31) where it covers a clip of S + 1 frames, else the generic kernel (contiguous tensors, any Cq and C,
    H + W + S - 1 <= 2048).  There is no backward: train with ``cca3d(..., causal=True)``.

    The caches are a ring of N = k_cache.shape[2] slots: ``frames`` (S, None: N) of them hold past frames, frame j (time
    order) in slot (head + j) % N.  The defaults are the caches in time order.  A stream over a window of W frames keeps a
    ring of W slots and overwrites the oldest frame's slot after each step (``CrissCrossAttention3D(..., window=W).step``):
    frame t, stepped with the last min(t, W) frames, is frame t of ``cca3d_forward(..., causal=True, window=W)``."""
    if torch.is_grad_enabled() and any(t.requires_grad for t in (q, k, v, k_cache, v_cache)):
        raise RuntimeError("ccnet_b200: cca3d_step has no backward (streaming inference); train with "
                           "cca3d(q, k, v, causal=True) on clips")
    _check_inputs(q, k, v)
    B, Cq, H, W = q.shape
    C = v.shape[1]
    if (k_cache.dim() != 5 or v_cache.dim() != 5 or tuple(k_cache.shape[:2]) != (B, Cq) or tuple(k_cache.shape[3:]) != (H, W)
            or tuple(v_cache.shape) != (B, C, k_cache.shape[2], H, W)):
        raise RuntimeError(f"ccnet_b200: expected k_cache [B,Cq,S,H,W] and v_cache [B,C,S,H,W] for q{tuple(q.shape)} "
                           f"v{tuple(v.shape)}, got {tuple(k_cache.shape)}, {tuple(v_cache.shape)}")
    if any(t.dtype != q.dtype or t.device != q.device for t in (k_cache, v_cache)):
        raise RuntimeError("ccnet_b200: k_cache, v_cache must match q, k, v in dtype and device")
    N = k_cache.shape[2]
    S = N if frames is None else int(frames)
    if not 0 <= S <= N or (N > 0 and not 0 <= head < N):
        raise ValueError(f"ccnet_b200: frames must be in [0, {N}] and head in [0, {N}), got frames={frames}, head={head}")
    det = _resolve_deterministic(deterministic)
    lib = capi.load()
    dt = _DTYPES[q.dtype]
    use_tc, flags, fmt = _plan(impl, det, _covered3d(capi.CCA_WS_FORWARD, q, v, S + 1), q, v)
    if use_tc and _upcast(q.dtype, H, W, det, S + 1):
        out32, lse = cca3d_step(q.float(), k.float(), v.float(), k_cache.float(), v_cache.float(), impl, det, S, head)
        return out32.to(q.dtype), lse
    cfmt = torch.channels_last_3d if use_tc else torch.contiguous_format
    q, k, v = (t.contiguous(memory_format=fmt) for t in (q, k, v))
    k_cache, v_cache = (t.contiguous(memory_format=cfmt) for t in (k_cache, v_cache))
    with torch.cuda.device(q.device):
        out = torch.empty_like(v, memory_format=fmt)
        lse = torch.empty((B, H, W), dtype=torch.float32, device=q.device)
        ws = _workspace(lib.cca_b200_workspace_bytes3d_step(B, Cq, C, S, H, W, dt, flags), q.device)
        rc = lib.cca_b200_forward3d_step_ring(q.data_ptr(), k.data_ptr(), v.data_ptr(), k_cache.data_ptr() if S else None,
                                              v_cache.data_ptr() if S else None, out.data_ptr(), lse.data_ptr(), ws.data_ptr(),
                                              ws.numel(), B, Cq, C, N, S, head, H, W, dt, flags, _stream_ptr(q.device))
        capi.check(rc, "cca_b200_forward3d_step_ring")
    return out, lse
