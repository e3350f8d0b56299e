"""GPU tests (H100: ``pytest -m gpu``) of criss-cross attention over clips (the 3D op): forward and backward against the fp64
oracle of tests/cca3d_oracle.py in fp32, bf16 and fp16 at the budgets of the 2D kernels, the T = 1 and H = 1 identities with
the 2D op, bit-reproducibility in deterministic mode, the CrissCrossAttention3D module, the C ABI's refusals and
torch.compile.  Each comparison prints one ``ERR {json}`` line (run with ``-s`` to see the measured errors)."""
import json

import pytest
import torch

import cca3d_oracle as O3
import f16_budget as fb
import tc_budget as tb

pytestmark = pytest.mark.gpu

T_MAX = 32
BF16_BUDGET = {n: 1e-2 for n in tb.TENSORS}


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _inputs(shape, dtype, seed, scale=0.7):
    B, Cq, C, T, H, W = shape
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Cq, T, H, W, generator=g) * scale
    k = torch.randn(B, Cq, T, H, W, generator=g) * scale
    v = torch.randn(B, C, T, H, W, generator=g)
    dout = torch.randn(B, C, T, H, W, generator=g)
    return tuple(t.to(dtype) for t in (q, k, v, dout))


def _reference(q, k, v, dout):
    q, k, v, dout = (t.double() for t in (q, k, v, dout))
    out, lse = O3.cca3d_forward(q, k, v)
    dq, dk, dv = O3.cca3d_backward(dout, q, k, v)
    return dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv)


def _run(q, k, v, dout, impl="auto", deterministic=None):
    from ccnet_b200 import cca3d_backward, cca3d_forward
    dev = _dev()
    q, k, v, dout = (t.to(dev) for t in (q, k, v, dout))
    out, lse = cca3d_forward(q, k, v, impl, deterministic)
    dq, dk, dv = cca3d_backward(dout, q, k, v, out, lse, impl, deterministic)
    torch.cuda.synchronize()
    return dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv)


def _check(got, ref, budget, what):
    errs = tb.check({n: t.cpu() for n, t in got.items()}, ref, budget, what)
    print("ERR", json.dumps(dict(what=what, err={n: float(f"{e:.2e}") for n, e in errs.items()})))
    return errs


BUDGETS = {torch.float32: tb.FP32_BUDGET, torch.bfloat16: BF16_BUDGET, torch.float16: fb.F16_BUDGET}
# (B, Cq, C, T, H, W)
SHAPES = [
    (1, 16, 64, 1, 5, 6),          # T = 1
    (1, 32, 64, 2, 7, 9),          # T = 2
    (2, 48, 128, 3, 9, 8),         # T = 3, B > 1
    (1, 64, 64, 4, 1, 11),         # H = 1
    (1, 16, 128, 5, 10, 1),        # W = 1
    (3, 32, 64, 8, 12, 10),        # B > 1
    (1, 64, 128, T_MAX, 6, 5),     # T at the bound
    (1, 16, 64, 9, 17, 9),         # T past the first register tier (8)
    (2, 32, 64, 17, 5, 7),         # T past the second tier (16)
    (1, 16, 64, 2, 113, 130),      # tiled lines
    (1, 48, 64, 3, 225, 20),       # tiled columns
]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
def test_forward_backward_vs_oracle(shape, dtype):
    """16-bit I/O on lines longer than 112 pixels runs on the fp32 kernels and is rounded once (as in 2D): fp16 lse is then
    held to the fp32 budget, as in tests/test_gpu_f16.py (the bf16x3 error of S reaches lse directly)"""
    budget = dict(BUDGETS[dtype])
    if dtype == torch.float16 and max(shape[4:]) > 112:
        budget["lse"] = tb.FP32_BUDGET["lse"]
    q, k, v, dout = _inputs(shape, dtype, seed=sum(shape))
    _check(_run(q, k, v, dout), _reference(q, k, v, dout), budget, f"{shape} {dtype}")


SIMT_BUDGETS = {torch.float32: tb.FP32_SIMT, torch.bfloat16: BF16_BUDGET, torch.float16: fb.F16_SIMT}
# shapes of the generic kernels: ragged channel counts, T past the tensor-core bound, a line over 896 pixels, H = 1, W = 1
SIMT_SHAPES = [
    (1, 8, 24, 3, 5, 6),
    (2, 5, 40, 1, 4, 7),
    (1, 16, 64, T_MAX + 1, 4, 3),
    (1, 3, 16, 2, 900, 2),
    (2, 7, 33, 4, 1, 9),
    (1, 12, 20, 5, 8, 1),
]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("shape", SIMT_SHAPES, ids=["x".join(map(str, s)) for s in SIMT_SHAPES])
def test_generic_kernels_vs_oracle(shape, dtype):
    """impl="simt" (NCDHW, any Cq and C) forward and backward against the fp64 oracle; "auto" picks the same kernels on
    shapes the tensor-core path does not cover, with the same bits"""
    from ccnet_b200.functional import tc3d_eligible
    q, k, v, dout = _inputs(shape, dtype, seed=sum(shape) + 1)
    got = _run(q, k, v, dout, impl="simt")
    assert got["out"].is_contiguous()
    _check(got, _reference(q, k, v, dout), SIMT_BUDGETS[dtype], f"simt {shape} {dtype}")
    if not tc3d_eligible(shape[0], shape[1], shape[2], *shape[3:], dtype):
        auto = _run(q, k, v, dout)
        assert all(torch.equal(auto[n], got[n]) for n in got)


def test_t_past_the_bound_falls_back_to_the_generic_kernels():
    """T = 33 with tensor-core channel counts: "auto" runs the generic kernels, "tc" refuses"""
    from ccnet_b200 import cca3d_forward
    from ccnet_b200.functional import tc3d_eligible
    assert tc3d_eligible(1, 16, 64, T_MAX, 4, 4, torch.float32) and not tc3d_eligible(1, 16, 64, T_MAX + 1, 4, 4, torch.float32)
    q, k, v, dout = _inputs((1, 16, 64, T_MAX + 1, 4, 4), torch.float32, seed=1)
    got = _run(q, k, v, dout)
    assert got["out"].is_contiguous()
    _check(got, _reference(q, k, v, dout), tb.FP32_SIMT, "T past the bound, auto")
    with pytest.raises(RuntimeError, match="do not cover"):
        cca3d_forward(q.cuda(), k.cuda(), v.cuda(), "tc")


@pytest.mark.parametrize("shape", [(2, 32, 64, 5, 9, 11), (1, 16, 64, T_MAX, 4, 6), (1, 16, 64, 2, 113, 20)],
                         ids=["small", "T32", "tiled"])
def test_tensor_core_and_generic_paths_agree(shape):
    """the composed tensor-core path and the independent generic kernels, fp32, within the sum of their budgets"""
    q, k, v, dout = _inputs(shape, torch.float32, seed=sum(shape) + 2)
    a, b = _run(q, k, v, dout, impl="tc"), _run(q, k, v, dout, impl="simt")
    errs = {n: tb.error(n, a[n], b[n].cpu().double()) for n in a}
    print("ERR", json.dumps(dict(what=f"tc vs simt {shape}", err=errs)))
    assert all(errs[n] <= tb.FP32_BUDGET[n] + tb.FP32_SIMT[n] for n in errs), errs


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["fp32", "bf16", "fp16"])
def test_t1_is_bitwise_the_2d_op(dtype):
    from ccnet_b200 import cca_backward, cca_forward
    q, k, v, dout = (t.cuda() for t in _inputs((2, 64, 128, 1, 20, 30), dtype, seed=7))
    g3 = _run(q, k, v, dout)
    q2, k2, v2, d2 = (t[:, :, 0] for t in (q, k, v, dout))
    out, lse = cca_forward(q2, k2, v2)
    dq, dk, dv = cca_backward(d2, q2, k2, v2, out, lse)
    for name, a, b in (("out", g3["out"], out), ("lse", g3["lse"], lse), ("dq", g3["dq"], dq), ("dk", g3["dk"], dk),
                       ("dv", g3["dv"], dv)):
        assert torch.equal(a[:, :, 0] if name != "lse" else a[:, 0], b), name


def test_h1_identity_agrees_with_both_2d_kernel_families():
    """H = 1: the 3D op is the 2D op on [B, C, T, W] (T as the column axis); the 2D tensor-core and generic kernels agree
    with it within their fp32 budgets"""
    from ccnet_b200 import cca_backward, cca_forward
    q, k, v, dout = (t.cuda() for t in _inputs((2, 32, 64, 9, 1, 14), torch.float32, seed=11))
    g3 = _run(q, k, v, dout)
    q2, k2, v2, d2 = (t[:, :, :, 0] for t in (q, k, v, dout))
    for impl, budget in (("tc", tb.FP32_BUDGET), ("simt", tb.FP32_SIMT)):
        out, lse = cca_forward(q2, k2, v2, impl)
        dq, dk, dv = cca_backward(d2, q2, k2, v2, out, lse, impl)
        ref = dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv)
        got = {n: (t[:, :, 0] if n == "lse" else t[:, :, :, 0]) for n, t in g3.items()}
        errs = {n: tb.error(n, got[n], ref[n].cpu().double()) for n in ref}
        print("ERR", json.dumps(dict(what=f"H=1 vs 2D {impl}", err=errs)))
        assert all(errs[n] <= tb.FP32_BUDGET[n] + budget[n] for n in errs), (impl, errs)


def test_deterministic_mode_is_bit_reproducible_on_tiled_lines():
    q, k, v, dout = _inputs((2, 16, 64, 3, 130, 113), torch.float32, seed=5)
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        a = _run(q, k, v, dout)
        b = _run(q, k, v, dout)
    finally:
        torch.use_deterministic_algorithms(was)
    assert all(torch.equal(a[n], b[n]) for n in a), [n for n in a if not torch.equal(a[n], b[n])]
    _check(a, _reference(q, k, v, dout), tb.FP32_BUDGET, "deterministic tiled")


# ---------------------------------------------------------------------------------------------------------------------
# the module
# ---------------------------------------------------------------------------------------------------------------------
def _module_pair(C, gamma, seed=0):
    from ccnet_b200 import CrissCrossAttention3D
    torch.manual_seed(seed)
    ref = O3.CrissCrossAttention3DOracle(C).double()
    with torch.no_grad():
        ref.gamma.fill_(gamma)
    m = CrissCrossAttention3D(C).cuda()
    m.load_state_dict({n: p.float() for n, p in ref.state_dict().items()})
    return m, ref


def _module_errors(m, ref, x, autocast=None, half=False):
    g = torch.randn_like(x)
    xd = x.cuda().requires_grad_(True) if not half else x.cuda().half().requires_grad_(True)
    if autocast is not None:
        with torch.autocast("cuda", dtype=autocast):
            y = m(xd)
    else:
        y = m(xd)
    (y.float() * g.cuda()).sum().backward()
    xr = x.double().requires_grad_(True)
    yr = ref(xr)
    (yr * g.double()).sum().backward()
    rel = lambda a, b: (a.detach().double().cpu() - b).abs().max().item() / max(1.0, b.abs().max().item())
    errs = dict(y=rel(y, yr.detach()), dx=rel(xd.grad, xr.grad))
    for (n, p), (_, pr) in zip(m.named_parameters(), ref.named_parameters()):
        errs[n] = rel(p.grad, pr.grad)
    return errs


@pytest.mark.parametrize("mode,tol", [("fp32", 1e-3), ("fp32-contiguous", 1e-3), ("autocast-fp16", 1e-2),
                                      ("autocast-bf16", 5e-2), ("half", 1e-2)])
def test_module_vs_fp64_oracle_module(mode, tol):
    torch.backends.cuda.matmul.allow_tf32 = False
    m, ref = _module_pair(128, 0.7)
    x = torch.randn(2, 128, 3, 9, 8)
    if mode == "half":
        m = m.half()
        x = x.half().float()                     # the oracle sees the same (rounded) input
        with torch.no_grad():
            for p, pr in zip(m.parameters(), ref.parameters()):
                pr.copy_(p.double())
    xin = x if mode == "fp32-contiguous" else x.contiguous(memory_format=torch.channels_last_3d)
    errs = _module_errors(m, ref, xin, autocast={"autocast-fp16": torch.float16, "autocast-bf16": torch.bfloat16}.get(mode),
                          half=mode == "half")
    print("ERR", json.dumps(dict(what=f"module {mode}", err={n: float(f"{e:.2e}") for n, e in errs.items()})))
    # The key bias gets no gradient in exact arithmetic (q . b_k is the same for all keys of a query, and the softmax ignores
    # it): its measured gradient is the rounding of a sum of per-pixel dk over all N pixels, which grows like sqrt(N).
    npix = x.shape[0] * x.shape[2] * x.shape[3] * x.shape[4]
    assert len(errs) == 9 and errs.pop("key_conv.bias") <= tol * npix ** 0.5, errs
    assert all(e <= tol for e in errs.values()), errs


def test_module_on_the_generic_kernels_vs_fp64_oracle_module():
    """in_dim = 64 (Cq = 8): stock Conv3d projections and the generic kernels"""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    m, ref = _module_pair(64, 0.7)
    errs = _module_errors(m, ref, torch.randn(2, 64, 3, 7, 6))
    print("ERR", json.dumps(dict(what="module generic", err={n: float(f"{e:.2e}") for n, e in errs.items()})))
    assert len(errs) == 9 and all(e <= 1e-4 for e in errs.values()), errs


def test_module_with_gamma_zero_returns_x():
    from ccnet_b200 import CrissCrossAttention3D
    m = CrissCrossAttention3D(128).cuda()
    x = torch.randn(1, 128, 4, 6, 7, device="cuda")
    assert torch.equal(m(x), x)


# ---------------------------------------------------------------------------------------------------------------------
# C ABI refusals, torch.compile
# ---------------------------------------------------------------------------------------------------------------------
def test_c_abi_refusals_leave_the_output_untouched():
    from ccnet_b200 import capi
    lib = capi.load()
    B, Cq, C, T, H, W = 1, 16, 64, 3, 6, 5
    dev = _dev()
    q = torch.randn(B, Cq, T, H, W, device=dev).contiguous(memory_format=torch.channels_last_3d)
    v = torch.randn(B, C, T, H, W, device=dev).contiguous(memory_format=torch.channels_last_3d)
    out = torch.full((B * C * T * H * W + 16,), 7.0, device=dev)
    lse = torch.full((B * T * H * W,), 7.0, device=dev)
    nhwc = capi.CCA_FLAG_NHWC
    nws = lib.cca_b200_workspace_bytes3d(capi.CCA_WS_FORWARD, B, Cq, C, T, H, W, capi.CCA_F32, nhwc)
    nws33 = lib.cca_b200_workspace_bytes3d(capi.CCA_WS_FORWARD, B, Cq, C, T_MAX + 1, H, W, capi.CCA_F32, nhwc)
    ws = torch.empty(max(nws, nws33), dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream().cuda_stream

    def call(qp, outp, nbytes, dims, flags):
        return lib.cca_b200_forward3d(qp, q.data_ptr(), v.data_ptr(), outp, lse.data_ptr(), ws.data_ptr(), nbytes, *dims,
                                      capi.CCA_F32, flags, st)
    dims = (B, Cq, C, T, H, W)
    assert call(q.data_ptr(), out.data_ptr(), nws, (B, Cq, C, 0, H, W), nhwc) == capi_status("INVALID")
    assert call(q.data_ptr(), out.data_ptr(), nws, (B, 8, C, T, H, W), nhwc | capi.CCA_FLAG_FORCE_TC) == capi_status("UNSUPPORTED")
    assert call(q.data_ptr(), out.data_ptr(), nws, dims, nhwc | capi.CCA_FLAG_FORCE_SIMT) == capi_status("UNSUPPORTED")
    assert call(q.data_ptr(), out.data_ptr(), nws - 16, dims, nhwc) == capi_status("WORKSPACE")
    assert call(q.data_ptr(), out.data_ptr() + 4, nws, dims, nhwc) == capi_status("INVALID")
    assert b"aligned" in lib.cca_b200_last_error()
    assert call(q.data_ptr(), out.data_ptr(), nws33, (B, Cq, C, T_MAX + 1, H, W), nhwc) == capi_status("UNSUPPORTED")
    assert call(q.data_ptr(), out.data_ptr(), 1 << 40, (B, Cq, C, T, 1500, 600), 0) == capi_status("UNSUPPORTED")  # > 2048 keys
    torch.cuda.synchronize()
    assert (out == 7.0).all() and (lse == 7.0).all()
    assert call(q.data_ptr(), out.data_ptr(), nws, dims, nhwc) == 0                                   # (the same call, valid)
    torch.cuda.synchronize()
    assert (out[:B * C * T * H * W] != 7.0).all() and (out[B * C * T * H * W:] == 7.0).all()


def test_c_abi_backward_refusals_leave_the_gradients_untouched():
    from ccnet_b200 import capi
    lib = capi.load()
    dev = _dev()
    st = torch.cuda.current_stream().cuda_stream
    nhwc, det = capi.CCA_FLAG_NHWC, capi.CCA_FLAG_DETERMINISTIC

    def tensors(B, Cq, C, T, H, W, dtype):
        mk = lambda c: torch.randn(B, c, T, H, W, device=dev).to(dtype).contiguous(memory_format=torch.channels_last_3d)
        q, k, v, g = mk(Cq), mk(Cq), mk(C), mk(C)
        from ccnet_b200 import cca3d_forward
        out, lse = cca3d_forward(q, k, v)
        grads = [torch.full_like(t, 7.0) for t in (q, k, v)]
        return q, k, v, g, out, lse, grads

    def call(ts, dims, dt, flags, nbytes=None, dq_off=0):
        q, k, v, g, out, lse, (dq, dk, dv) = ts
        need = lib.cca_b200_workspace_bytes3d(capi.CCA_WS_BACKWARD, *dims, dt, flags)
        ws = torch.empty(need + 64, dtype=torch.uint8, device=dev)
        return lib.cca_b200_backward3d(g.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(),
                                       dq.data_ptr() + dq_off, dk.data_ptr(), dv.data_ptr(), ws.data_ptr(),
                                       need if nbytes is None else nbytes, *dims, dt, flags, st)

    dims = (1, 16, 64, 3, 6, 5)
    ts = tensors(*dims, torch.float32)
    assert call(ts, (1, 16, 64, 0, 6, 5), capi.CCA_F32, nhwc) == capi_status("INVALID")
    assert call(ts, dims, capi.CCA_F32, nhwc, nbytes=16) == capi_status("WORKSPACE")
    assert call(ts, (1, 8, 64, 3, 6, 5), capi.CCA_F32, nhwc | capi.CCA_FLAG_FORCE_TC) == capi_status("UNSUPPORTED")
    assert call(ts, dims, capi.CCA_F32, nhwc | capi.CCA_FLAG_FORCE_SIMT) == capi_status("UNSUPPORTED")
    assert call(ts, dims, capi.CCA_F32, nhwc, dq_off=4) == capi_status("INVALID")
    assert b"aligned" in lib.cca_b200_last_error()
    # 16-bit I/O with the deterministic flag on lines longer than one tile: no planes mode for it
    tiled = (1, 16, 64, 2, 113, 20)
    th = tensors(*tiled, torch.bfloat16)
    assert call(th, tiled, capi.CCA_BF16, nhwc | det) == capi_status("UNSUPPORTED")
    assert b"DETERMINISTIC" in lib.cca_b200_last_error()
    torch.cuda.synchronize()
    for _, _, _, _, _, _, grads in (ts, th):
        assert all((t == 7.0).all() for t in grads)
    assert call(ts, dims, capi.CCA_F32, nhwc) == 0                          # (valid)
    torch.cuda.synchronize()
    assert not any((t == 7.0).all() for t in ts[6])


def capi_status(name):
    return {"INVALID": -1, "UNSUPPORTED": -2, "WORKSPACE": -3}[name]


def test_torch_compile_fullgraph():
    import ccnet_b200  # noqa: F401
    q, k, v, _ = (t.cuda() for t in _inputs((1, 16, 64, 3, 8, 9), torch.float32, seed=3))

    def f(q, k, v):
        out, lse = torch.ops.cca.forward3d(q, k, v)
        return out * 2, lse

    fc = torch.compile(f, fullgraph=True)
    a, la = fc(q, k, v)
    b, lb = f(q, k, v)
    assert torch.equal(a, b) and torch.equal(la, lb)
