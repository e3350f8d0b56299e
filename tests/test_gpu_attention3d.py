"""H100 tests (``pytest -m gpu``) of the attention map of criss-cross attention over clips: both kernel families against the
fp64 oracle within budgets derived by emulation (tests/attn3d_budget.py) over the shapes of tests/test_gpu_cca3d.py, their
agreement, the T = 1 identity with the 2D map, the fallback past T = 32, determinism, the C ABI's refusals, views at odd
offsets, a map past 2^31 elements, the CrissCrossAttention3D module and the torch.ops registration."""
import json

import pytest
import torch

import attn3d_budget as A3
import ccnet_b200
from ccnet_b200 import capi
from ccnet_b200.functional import (_upcast, attention3d_tc_eligible, cca3d_attention_backward, cca3d_attention_forward,
                                   cca_attention_backward, cca_attention_forward)

pytestmark = pytest.mark.gpu
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
T_MAX = 32
# (B, Cq, C, T, H, W) of tests/test_gpu_cca3d.py (C unused by the map)
SHAPES = [(1, 16, 64, 1, 5, 6), (1, 32, 64, 2, 7, 9), (2, 48, 128, 3, 9, 8), (1, 64, 64, 4, 1, 11), (1, 16, 128, 5, 10, 1),
          (3, 32, 64, 8, 12, 10), (1, 64, 128, T_MAX, 6, 5), (1, 16, 64, 9, 17, 9), (2, 32, 64, 17, 5, 7),
          (1, 16, 64, 2, 113, 130), (1, 48, 64, 3, 225, 20)]


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _inputs(shape, dtype, seed, scale=0.7):
    B, Cq, _, T, H, W = shape
    g = torch.Generator().manual_seed(seed)
    q, k = ((torch.randn(B, Cq, T, H, W, generator=g) * scale).to(dtype) for _ in range(2))
    da = torch.randn(B, T, H, W, H + W + T, generator=g)
    return q, k, da


def _run(q, k, da, impl="auto", deterministic=None):
    dev = _dev()
    qd, kd = q.to(dev), k.to(dev)
    attn = cca3d_attention_forward(qd, kd, impl, deterministic)
    dq, dk = cca3d_attention_backward(da.to(dev), attn, qd, kd, impl, deterministic)
    torch.cuda.synchronize()
    return dict(attn=attn, dq=dq, dk=dk)


@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).split(".")[-1])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_map_and_gradients_match_the_oracle(shape, dtype, impl):
    B, Cq, _, T, H, W = shape
    q, k, da = _inputs(shape, dtype, seed=sum(shape))
    native = impl == "simt" or not _upcast(dtype, H, W, False, T)
    ref, emu = A3.reference(q, k, da), A3.emulate(q, k, da, dtype, native)
    bud = A3.budget(emu, ref, dtype)
    got = _run(q, k, da, impl)
    a = got["attn"]
    assert a.dtype == torch.float32 and a.is_contiguous() and tuple(a.shape) == (B, T, H, W, H + W + T)
    assert got["dq"].dtype == dtype and got["dk"].dtype == dtype
    if impl == "tc":
        assert got["dq"].is_contiguous(memory_format=torch.channels_last_3d)
    errs = A3.check(got, ref, bud, (shape, dtype, impl))
    print("ERR", json.dumps(dict(what=f"{shape} {dtype} {impl}", err={n: float(f"{e:.2e}") for n, e in errs.items()})))
    assert a.min().item() >= 0
    assert (a.sum(-1) - 1).abs().max().item() < 1e-5 * (H + W + T) ** 0.5 + 1e-5
    assert a[..., :H].diagonal(dim1=2, dim2=4).abs().max().item() == 0
    assert a[..., H + W:].diagonal(dim1=1, dim2=4).abs().max().item() == 0


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).split(".")[-1])
def test_tensor_core_and_generic_kernels_agree(dtype):
    q, k, da = _inputs((2, 32, 0, 6, 13, 11), dtype, seed=11)
    tc, simt = _run(q, k, da, "tc"), _run(q, k, da, "simt")
    ref = A3.reference(q, k, da)
    bud = A3.budget(A3.emulate(q, k, da, dtype, not _upcast(dtype, 13, 11, False, 6)), ref, dtype)
    for n in tc:
        assert A3.error(tc[n], simt[n].cpu().double()) <= 2 * bud[n], n


@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).split(".")[-1])
@pytest.mark.parametrize("shape", [(2, 16, 9, 7), (1, 32, 113, 130)], ids=lambda s: "x".join(map(str, s)))
def test_t1_is_the_2d_map_to_the_bit(shape, dtype, impl):
    """T = 1: attn[..., :H+W] and dq, dk are the 2D map's bits (negative zeros included), attn[..., H+W] is 0.  On tiled
    lines both run in the deterministic mode: otherwise their dq, dk reduce-adds land in no fixed order, in 2D as well."""
    dev = _dev()
    B, Cq, H, W = shape
    det = max(H, W) > 112
    g = torch.Generator().manual_seed(12)
    q, k = ((torch.randn(B, Cq, H, W, generator=g) * 0.7).to(dtype).to(dev) for _ in range(2))
    da = torch.randn(B, H, W, H + W + 1, generator=g).to(dev)
    a2 = cca_attention_forward(q, k, impl, det)
    a3 = cca3d_attention_forward(q.unsqueeze(2), k.unsqueeze(2), impl, det)
    assert torch.equal(a3[:, 0, ..., :H + W], a2) and not a3[..., H + W].any()
    g2 = cca_attention_backward(da[..., :H + W].contiguous(), a2, q, k, impl, det)
    g3 = cca3d_attention_backward(da.unsqueeze(1), a3, q.unsqueeze(2), k.unsqueeze(2), impl, det)
    for x2, x3 in zip(g2, g3):
        x3 = x3[:, :, 0]
        assert torch.equal(x3, x2) and torch.equal(torch.signbit(x3), torch.signbit(x2))


def test_t_past_the_bound_falls_back_to_the_generic_kernels():
    assert attention3d_tc_eligible(1, 16, T_MAX, 4, 4, torch.float32)
    assert not attention3d_tc_eligible(1, 16, T_MAX + 1, 4, 4, torch.float32)
    q, k, da = _inputs((1, 16, 0, T_MAX + 1, 4, 4), torch.float32, seed=13)
    auto, simt = _run(q, k, da), _run(q, k, da, "simt")
    assert all(torch.equal(auto[n], simt[n]) for n in auto) and auto["dq"].is_contiguous()
    with pytest.raises(RuntimeError, match="do not cover"):
        _run(q, k, da, "tc")


@pytest.mark.parametrize("shape", [(2, 32, 0, 3, 129, 129), (1, 16, 0, 4, 113, 200)], ids=lambda s: "x".join(map(str, s)))
def test_deterministic_mode_is_bit_reproducible(shape, monkeypatch):
    q, k, da = _inputs(shape, torch.float32, seed=14)
    runs = [_run(q, k, da, deterministic=True) for _ in range(3)]
    from ccnet_b200 import functional
    monkeypatch.setattr(functional, "deterministic_workspace_cap", 1)          # one sample per call
    runs.append(_run(q, k, da, deterministic=True))
    for r in runs[1:]:
        assert all(torch.equal(runs[0][n], r[n]) for n in r)


@pytest.mark.parametrize("dtype", [capi.CCA_BF16, capi.CCA_F16])
def test_16bit_deterministic_tiled_backward_is_refused_and_leaves_outputs_untouched(dtype):
    dev = _dev()
    lib = capi.load()
    B, Cq, T, H, W = 1, 16, 2, 129, 129
    q = torch.zeros(B, Cq, T, H, W, dtype=torch.float16, device=dev).contiguous(memory_format=torch.channels_last_3d)
    a = torch.zeros(B, T, H, W, H + W + T, device=dev)
    dq = torch.full_like(q, 7.0)
    flags = capi.CCA_FLAG_NHWC | capi.CCA_FLAG_DETERMINISTIC
    ws = torch.empty(lib.cca_b200_attention_workspace_bytes3d(1, B, Cq, T, H, W, dtype, flags), dtype=torch.uint8, device=dev)
    rc = lib.cca_b200_attention_backward3d(a.data_ptr(), a.data_ptr(), q.data_ptr(), q.data_ptr(), dq.data_ptr(), dq.data_ptr(),
                                           ws.data_ptr(), ws.numel(), B, Cq, T, H, W, dtype, flags, None)
    torch.cuda.synchronize()
    assert rc == -2 and b"DETERMINISTIC" in lib.cca_b200_last_error()
    assert (dq == 7).all()


def test_refusals_leave_sentinel_outputs_untouched():
    dev = _dev()
    lib = capi.load()
    B, Cq, T, H, W = 1, 16, 3, 9, 9
    q = torch.randn(B, Cq, T, H, W, device=dev).contiguous(memory_format=torch.channels_last_3d)
    attn = torch.full((B, T, H, W, H + W + T), -5.0, device=dev)
    dq = torch.full_like(q, 3.0)
    nhwc, both = capi.CCA_FLAG_NHWC, capi.CCA_FLAG_FORCE_SIMT | capi.CCA_FLAG_FORCE_TC
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=dev)
    for flags, nbytes in ((both, ws.numel()), (nhwc, 16), (nhwc | capi.CCA_FLAG_FORCE_SIMT, ws.numel())):
        rc = lib.cca_b200_attention_forward3d(q.data_ptr(), q.data_ptr(), attn.data_ptr(), ws.data_ptr(), nbytes,
                                              B, Cq, T, H, W, capi.CCA_F32, flags, None)
        assert rc < 0
        rc = lib.cca_b200_attention_backward3d(attn.data_ptr(), attn.data_ptr(), q.data_ptr(), q.data_ptr(), dq.data_ptr(),
                                               dq.data_ptr(), ws.data_ptr(), nbytes, B, Cq, T, H, W, capi.CCA_F32, flags, None)
        assert rc < 0
    torch.cuda.synchronize()
    assert (attn == -5).all() and (dq == 3).all()


@pytest.mark.parametrize("impl", ["tc", "simt"])
def test_backward_takes_attn_and_dattn_at_any_float_offset(impl):
    dev = _dev()
    q, k, da = _inputs((2, 32, 0, 3, 17, 13), torch.float32, seed=15)     # H + W + T odd
    q, k, da = q.to(dev), k.to(dev), da.to(dev)
    attn = cca3d_attention_forward(q, k, impl)
    ref = cca3d_attention_backward(da, attn, q, k, impl)
    odd = lambda t: torch.empty(t.numel() + 1, device=dev)[1:].view(t.shape).copy_(t)
    for a, d in ((attn, odd(da)), (odd(attn), da), (odd(attn), odd(da))):
        assert (a.data_ptr() | d.data_ptr()) % 8 == 4
        got = cca3d_attention_backward(d, a, q, k, impl)
        assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])


def test_map_past_2_31_elements_matches_the_oracle_on_sampled_pixels():
    dev = _dev()
    B, Cq, T, H, W = 2, 16, 4, 512, 512
    assert B * T * H * W * (H + W + T) > 2 ** 31
    g = torch.Generator(device=dev).manual_seed(16)
    q, k = ((torch.randn(B, Cq, T, H, W, device=dev, generator=g) * 0.5).contiguous(memory_format=torch.channels_last_3d)
            for _ in range(2))
    attn = cca3d_attention_forward(q, k)
    pix = ((1, 3, 511, 511), (1, 2, 400, 3), (0, 0, 0, 0), (1, 1, 256, 300))
    qd, kd = q.double(), k.double()

    def row(b, t, h, w):
        qv = qd[b, :, t, h, w]
        col, rw, tm = qv @ kd[b, :, t, :, w], qv @ kd[b, :, t, h, :], qv @ kd[b, :, :, h, w]
        col[h], tm[t] = float("-inf"), float("-inf")
        return torch.softmax(torch.cat([col, rw, tm]), 0)

    for b, t, h, w in pix:
        assert (attn[b, t, h, w].double() - row(b, t, h, w)).abs().max().item() < 1e-5
    dattn = torch.randn(attn.shape, device=dev, generator=g)
    dq, dk = cca3d_attention_backward(dattn, attn, q, k)
    ds = lambda a, d: a.double() * (d.double() - (a.double() * d.double()).sum(-1, keepdim=True))
    for b, t, h, w in pix:
        s = ds(attn[b, t, h, w], dattn[b, t, h, w])
        s[h], s[H + W + t] = 0, 0
        ref = kd[b, :, t, :, w] @ s[:H] + kd[b, :, t, h, :] @ s[H:H + W] + kd[b, :, :, h, w] @ s[H + W:]
        assert (dq[b, :, t, h, w].double() - ref).abs().max().item() <= 1e-4 * max(1.0, ref.abs().max().item())
        # the same pixel as a key: column queries (t, i, w), row queries (t, h, j), time queries (s, h, w)
        sc = ds(attn[b, t, :, w], dattn[b, t, :, w])[:, h]
        sc[h] = 0
        sr = ds(attn[b, t, h], dattn[b, t, h])[:, H + w]
        st = ds(attn[b, :, h, w], dattn[b, :, h, w])[:, H + W + t]
        st[t] = 0
        ref = qd[b, :, t, :, w] @ sc + qd[b, :, t, h, :] @ sr + qd[b, :, :, h, w] @ st
        assert (dk[b, :, t, h, w].double() - ref).abs().max().item() <= 1e-4 * max(1.0, ref.abs().max().item())


def _oracle_module(C, dtype=torch.float64):
    import cca3d_oracle as O3
    torch.manual_seed(17)
    ref = O3.CrissCrossAttention3DOracle(C)
    with torch.no_grad():
        ref.gamma.fill_(0.6)
    return ref


@pytest.mark.parametrize("C,impl", [(64, "auto"), (128, "auto"), (24, "auto"), (64, "simt")])
def test_return_attention_leaves_y_and_its_gradients_unchanged(C, impl):
    dev = _dev()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        m = ccnet_b200.CrissCrossAttention3D(C, impl).to(dev)
        m.load_state_dict(_oracle_module(C).state_dict())
        x = torch.randn(2, C, 3, 9, 11, device=dev)
        y0 = m(x)
        y0.square().sum().backward()
        g0 = [p.grad.clone() for p in m.parameters()]
        m.zero_grad()
        y1, a = m(x, return_attention=True)
        assert torch.equal(y0, y1) and a.shape == (2, 3, 9, 11, 23)
        y1.square().sum().backward()
        assert all(torch.equal(p.grad, g) for p, g in zip(m.parameters(), g0))
    finally:
        torch.use_deterministic_algorithms(False)


@pytest.mark.parametrize("C,impl,autocast,tol", [(128, "auto", None, 1e-5), (128, "auto", torch.float16, 2e-2),
                                                 (128, "auto", torch.bfloat16, 5e-2), (24, "simt", None, 1e-5)])
def test_module_map_and_gradients_match_the_oracle_module(C, impl, autocast, tol):
    dev = _dev()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    ref = _oracle_module(C)
    m = ccnet_b200.CrissCrossAttention3D(C, impl).to(dev)
    m.load_state_dict(ref.state_dict())
    x = torch.randn(2, C, 4, 10, 9)
    r = torch.randn(2, 4, 10, 9, 23)
    xd = x.to(dev).requires_grad_(True)
    with torch.autocast("cuda", dtype=autocast or torch.float16, enabled=autocast is not None):
        _, a = m(xd, return_attention=True)
    assert a.dtype == torch.float32
    (a * r.to(dev)).sum().backward()
    r64 = ref.double()
    xr = x.double().requires_grad_(True)
    ar = A3.attention_map3d(r64.query_conv(xr), r64.key_conv(xr))
    (ar * r.double()).sum().backward()
    rel = lambda got, want: (got.detach().cpu().double() - want).abs().max().item() / max(1.0, want.abs().max().item())
    assert rel(a, ar.detach()) < tol
    assert rel(xd.grad, xr.grad) < 10 * tol
    for n in ("query_conv.weight", "key_conv.weight", "query_conv.bias", "key_conv.bias"):
        assert rel(dict(m.named_parameters())[n].grad, dict(r64.named_parameters())[n].grad) < 10 * tol, n


def test_torch_ops_opcheck_and_compile_without_graph_break():
    dev = _dev()
    q, k, da = (t.to(dev) for t in _inputs((2, 16, 0, 3, 9, 11), torch.float32, seed=18))
    q, k = (t.contiguous(memory_format=torch.channels_last_3d) for t in (q, k))
    torch.library.opcheck(torch.ops.cca.attention3d.default, (q, k), test_utils=("test_schema", "test_faketensor"))
    torch.library.opcheck(torch.ops.cca.attention3d.default, (q.clone().requires_grad_(True), k.clone().requires_grad_(True)),
                          test_utils=("test_autograd_registration",))
    a = torch.ops.cca.attention3d(q, k)
    torch.library.opcheck(torch.ops.cca.attention3d_backward.default, (da, a, q, k), test_utils=("test_schema", "test_faketensor"))
    assert torch.equal(a, ccnet_b200.cca3d_attention(q, k))
    m = ccnet_b200.CrissCrossAttention3D(128).to(dev)
    x = torch.randn(2, 128, 3, 9, 11, device=dev)
    _, a0 = m(x, return_attention=True)

    def step_map(x):                         # what return_attention adds to the step: the convs and the map op
        return torch.ops.cca.attention3d(m.query_conv(x), m.key_conv(x), m.impl)
    a1 = torch.compile(step_map, fullgraph=True)(x)
    assert torch.allclose(a0, a1, atol=1e-6)
