"""GPU tests (H100: ``pytest -m gpu``) of causal criss-cross attention over clips (CCA_FLAG_CAUSAL) and its streaming step:
the causal forward, backward, map and map backward of both kernel families against the fp64 oracle of
tests/cca3d_causal_oracle.py in fp32, bf16 and fp16 at the budgets of the bidirectional op; frame 0 against the 2D op; the
deterministic mode; the step against the causal clip forward (bit for bit on the fp32 tensor-core path); the module's step
loop; torch.compile.  Each comparison prints one ``ERR {json}`` line (run with ``-s``)."""
import json

import pytest
import torch

import cca3d_causal_oracle as OC
import f16_budget as fb
import tc_budget as tb

pytestmark = pytest.mark.gpu

BF16_BUDGET = {n: 1e-2 for n in tb.TENSORS}
BUDGETS = {torch.float32: tb.FP32_BUDGET, torch.bfloat16: BF16_BUDGET, torch.float16: fb.F16_BUDGET}
SIMT_BUDGETS = {torch.float32: tb.FP32_SIMT, torch.bfloat16: BF16_BUDGET, torch.float16: fb.F16_SIMT}
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
IDS = ["fp32", "bf16", "fp16"]


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
    out, lse = OC.cca3d_causal_forward(q, k, v)
    dq, dk, dv = OC.cca3d_causal_backward(dout, q, k, v)
    return dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv)


def _run(q, k, v, dout, impl="auto", deterministic=None):
    from ccnet_b200 import cca3d_backward, cca3d_forward
    q, k, v, dout = (t.cuda() for t in (q, k, v, dout))
    out, lse = cca3d_forward(q, k, v, impl, deterministic, causal=True)
    dq, dk, dv = cca3d_backward(dout, q, k, v, out, lse, impl, deterministic, causal=True)
    torch.cuda.synchronize()
    return dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv)


def _check(got, ref, budget, what):
    errs = tb.check({n: t.cpu() for n, t in got.items()}, ref, budget, what)
    print("ERR", json.dumps(dict(what=what, err={n: float(f"{e:.2e}") for n, e in errs.items()})))
    return errs


# (B, Cq, C, T, H, W): T in {1, 2, 5, 8, 9, 16, 17, 32}, Cq in {16, 48, 64}, one-tile and tiled lines
SHAPES = [
    (1, 16, 64, 1, 5, 6),
    (2, 48, 128, 2, 9, 8),
    (1, 64, 64, 5, 7, 11),
    (2, 16, 64, 8, 6, 5),
    (1, 48, 64, 9, 5, 7),
    (1, 64, 128, 16, 4, 6),
    (1, 16, 64, 17, 5, 4),
    (1, 16, 64, 32, 4, 5),
    (1, 16, 64, 2, 129, 20),
]
SIDS = ["x".join(map(str, s)) for s in SHAPES]


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("shape", SHAPES, ids=SIDS)
def test_causal_forward_backward_vs_oracle(shape, dtype):
    budget = dict(BUDGETS[dtype])
    if dtype == torch.float16 and max(shape[4:]) > 112:
        budget["lse"] = tb.FP32_BUDGET["lse"]
    q, k, v, dout = _inputs(shape, dtype, seed=sum(shape))
    ref = _reference(q, k, v, dout)
    _check(_run(q, k, v, dout), ref, budget, f"tc {shape} {dtype}")
    _check(_run(q, k, v, dout, impl="simt"), ref, SIMT_BUDGETS[dtype], f"simt {shape} {dtype}")


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("shape", [SHAPES[1], SHAPES[4], SHAPES[7], SHAPES[8]], ids=[SIDS[1], SIDS[4], SIDS[7], SIDS[8]])
def test_causal_map_and_its_backward_vs_oracle(shape, dtype):
    """the map (time entries s >= t exactly 0) and dq, dk of both families; the map in fp32 is held to the forward's out
    budget of its family, dq and dk to the op's dq, dk budgets"""
    from ccnet_b200.functional import cca3d_attention_backward, cca3d_attention_forward
    B, Cq, C, T, H, W = shape
    q, k, _, _ = _inputs(shape, dtype, seed=sum(shape) + 3)
    g = torch.Generator().manual_seed(5)
    dattn = torch.randn(B, T, H, W, H + W + T, generator=g)
    a_ref = OC.cca3d_causal_attention(q.double(), k.double())
    dq_ref, dk_ref = OC.cca3d_causal_attention_backward(dattn.double(), q.double(), k.double())
    mask = OC.time_mask(T).view(1, T, 1, 1, T).expand(B, T, H, W, T)
    for impl, budgets in (("auto", BUDGETS), ("simt", SIMT_BUDGETS)):
        qc, kc = q.cuda(), k.cuda()
        attn = cca3d_attention_forward(qc, kc, impl, causal=True)
        dq, dk = cca3d_attention_backward(dattn.cuda(), attn, qc, kc, impl, causal=True)
        assert (attn[..., H + W:].cpu()[mask] == 0).all()
        errs = dict(attn=tb.error("out", attn.cpu(), a_ref), dq=tb.error("dq", dq.cpu(), dq_ref), dk=tb.error("dk", dk.cpu(), dk_ref))
        print("ERR", json.dumps(dict(what=f"map {impl} {shape} {dtype}", err=errs)))
        b = budgets[dtype]
        assert errs["attn"] <= max(b["out"], 1e-2 if dtype != torch.float32 else 0) and errs["dq"] <= b["dq"] and errs["dk"] <= b["dk"], errs


def test_generic_backward_past_the_tensor_core_bound():
    """T = 40, which only the generic kernels take: pins the transposed time gather of dk and dv"""
    shape = (1, 8, 24, 40, 3, 4)
    q, k, v, dout = _inputs(shape, torch.float32, seed=40)
    got = _run(q, k, v, dout)
    assert got["out"].is_contiguous()
    _check(got, _reference(q, k, v, dout), tb.FP32_SIMT, "simt T=40")


def test_frame_0_is_bitwise_the_2d_op():
    from ccnet_b200 import cca_forward, cca3d_backward, cca3d_forward, cca_backward
    q, k, v, dout = (t.cuda() for t in _inputs((2, 64, 128, 4, 20, 30), torch.float32, seed=7))
    out, lse = cca3d_forward(q, k, v, causal=True)
    o2, l2 = cca_forward(q[:, :, 0], k[:, :, 0], v[:, :, 0])
    assert torch.equal(out[:, :, 0], o2) and torch.equal(lse[:, 0], l2)
    dq, _, _ = cca3d_backward(dout, q, k, v, out, lse, causal=True)
    dq2, _, _ = cca_backward(dout[:, :, 0], q[:, :, 0], k[:, :, 0], v[:, :, 0], o2, l2)
    assert torch.equal(dq[:, :, 0], dq2)                   # (frame 0 has no time key: its dq gets +0 from the time pass)


def test_deterministic_mode_is_bit_reproducible():
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for shape in ((2, 16, 64, 3, 130, 113), (1, 32, 64, 6, 9, 10)):
            q, k, v, dout = _inputs(shape, torch.float32, seed=5)
            a, b = _run(q, k, v, dout), _run(q, k, v, dout)
            assert all(torch.equal(a[n], b[n]) for n in a), (shape, [n for n in a if not torch.equal(a[n], b[n])])
            _check(a, _reference(q, k, v, dout), tb.FP32_BUDGET, f"deterministic {shape}")
    finally:
        torch.use_deterministic_algorithms(was)


# ---------------------------------------------------------------------------------------------------------------------
# the streaming step
# ---------------------------------------------------------------------------------------------------------------------
def _step_vs_clip(shape, dtype, impl, bitwise, deterministic=None):
    from ccnet_b200 import cca3d_forward, cca3d_step
    q, k, v, _ = (t.cuda() for t in _inputs(shape, dtype, seed=sum(shape) + 11))
    T = shape[3]
    out, lse = cca3d_forward(q, k, v, impl, deterministic, causal=True)
    ref = OC.cca3d_causal_forward(q.double().cpu(), k.double().cpu(), v.double().cpu())
    for S in range(T):
        so, sl = cca3d_step(q[:, :, S], k[:, :, S], v[:, :, S], k[:, :, :S], v[:, :, :S], impl, deterministic)
        if bitwise:
            assert torch.equal(so, out[:, :, S]) and torch.equal(sl, lse[:, S]), (shape, S)
        errs = dict(out=tb.error("out", so.cpu(), ref[0][:, :, S]), lse=tb.error("lse", sl.cpu(), ref[1][:, S]))
        budget = (BUDGETS if impl != "simt" else SIMT_BUDGETS)[dtype]
        assert errs["out"] <= budget["out"] and errs["lse"] <= max(budget["lse"], tb.FP32_BUDGET["lse"]), (shape, S, errs)
    print("ERR", json.dumps(dict(what=f"step {impl} {shape} {dtype}", err=errs)))


@pytest.mark.parametrize("shape", [(2, 16, 64, 6, 9, 8), (1, 64, 128, 9, 7, 11), (1, 48, 64, 3, 129, 20)],
                         ids=["small", "T9", "tiled"])
def test_step_frame_by_frame_is_bitwise_the_causal_clip_forward(shape):
    _step_vs_clip(shape, torch.float32, "tc", bitwise=max(shape[4:]) <= 112)


def test_step_deterministic_on_tiled_lines_is_bitwise_the_causal_clip_forward():
    _step_vs_clip((1, 16, 64, 3, 20, 130), torch.float32, "tc", bitwise=True, deterministic=True)


def test_step_s31_and_s0():
    _step_vs_clip((1, 16, 64, 32, 4, 5), torch.float32, "tc", bitwise=True)


@pytest.mark.parametrize("shape", [(1, 8, 24, 5, 6, 7), (2, 16, 64, 4, 9, 8)], ids=["ragged", "tc-shape"])
def test_generic_step_is_bitwise_the_generic_causal_clip_forward(shape):
    _step_vs_clip(shape, torch.float32, "simt", bitwise=True)


def test_step_tensor_core_coverage_ends_at_31_cached_frames():
    """S = 31 runs on the tensor cores (channels-last out), S = 32 on the generic kernel (contiguous out); the C ABI refuses
    FORCE_TC at S = 32 before any launch and leaves out untouched"""
    from ccnet_b200 import capi, cca3d_step
    q, k, v, _ = (t.cuda() for t in _inputs((1, 16, 64, 33, 5, 6), torch.float32, seed=33))
    for S, cl in ((31, True), (32, False)):
        out, _ = cca3d_step(q[:, :, S], k[:, :, S], v[:, :, S], k[:, :, :S], v[:, :, :S])
        assert out.is_contiguous(memory_format=torch.channels_last) == cl and out.is_contiguous() != cl, S
    lib = capi.load()
    fl = capi.CCA_FLAG_NHWC | capi.CCA_FLAG_FORCE_TC
    qf, kf, vf = (t[:, :, 32].contiguous(memory_format=torch.channels_last) for t in (q, k, v))
    kc, vc = (t[:, :, :32].contiguous(memory_format=torch.channels_last_3d) for t in (k, v))
    out = torch.full_like(vf, 7.0)
    lse = torch.full((1, 5, 6), 7.0, device="cuda")
    nws = lib.cca_b200_workspace_bytes3d_step(1, 16, 64, 32, 5, 6, capi.CCA_F32, fl)
    ws = torch.empty(nws, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    rc = lib.cca_b200_forward3d_step(qf.data_ptr(), kf.data_ptr(), vf.data_ptr(), kc.data_ptr(), vc.data_ptr(), out.data_ptr(),
                                     lse.data_ptr(), ws.data_ptr(), nws, 1, 16, 64, 32, 5, 6, capi.CCA_F32, fl, st)
    torch.cuda.synchronize()
    assert rc == -2 and (out == 7.0).all() and (lse == 7.0).all()
    rc = lib.cca_b200_forward3d_step(qf.data_ptr(), kf.data_ptr(), vf.data_ptr(), kc.data_ptr(), vc.data_ptr(), out.data_ptr(),
                                     lse.data_ptr(), ws.data_ptr(), nws, 1, 16, 64, 31, 5, 6, capi.CCA_F32, fl, st)
    torch.cuda.synchronize()
    assert rc == 0 and not (out == 7.0).any()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_step_with_16bit_io(dtype):
    _step_vs_clip((2, 32, 64, 5, 9, 10), dtype, "auto", bitwise=False)
    _step_vs_clip((1, 8, 24, 4, 6, 7), dtype, "simt", bitwise=False)


# ---------------------------------------------------------------------------------------------------------------------
# the module
# ---------------------------------------------------------------------------------------------------------------------
def _causal_module(C, gamma=0.7, seed=0):
    from ccnet_b200 import CrissCrossAttention3D
    torch.manual_seed(seed)
    m = CrissCrossAttention3D(C, causal=True).cuda()
    with torch.no_grad():
        m.gamma.fill_(gamma)
    return m


@pytest.mark.parametrize("C", [128, 64], ids=["tc", "generic"])
def test_module_step_loop_equals_the_causal_forward(C):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    m = _causal_module(C)
    x = torch.randn(2, C, 6, 9, 8, device="cuda")
    with torch.no_grad():
        y = m(x)
        state, ys = None, []
        for t in range(6):
            yt, state = m.step(x[:, :, t], state)
            ys.append(yt)
        err = (torch.stack(ys, 2) - y).abs().max().item()
        # sliding window of max_frames + 1 = 4 frames
        state, errw = None, 0.0
        for t in range(6):
            yt, state = m.step(x[:, :, t], state, max_frames=3)
            assert state[0].shape[2] == min(t + 1, 3)
            w0 = max(0, t - 3)
            errw = max(errw, (yt - m(x[:, :, w0:t + 1])[:, :, -1]).abs().max().item())
    print("ERR", json.dumps(dict(what=f"module step C={C}", err=err, window=errw)))
    assert err <= 1e-4 and errw <= 1e-4, (err, errw)


def test_module_causal_attention_and_gradients():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    m = _causal_module(128)
    ref = OC.CausalCrissCrossAttention3DOracle(128).double()
    ref.load_state_dict({n: p.detach().double().cpu() for n, p in m.state_dict().items()})
    x = torch.randn(2, 128, 4, 7, 6)
    xd = x.cuda().requires_grad_(True)
    y, attn = m(xd, return_attention=True)
    g = torch.randn_like(x)
    ga = torch.randn(*attn.shape)
    ((y * g.cuda()).sum() + (attn * ga.cuda()).sum()).backward()
    xr = x.double().requires_grad_(True)
    yr = ref(xr)
    ar = OC.cca3d_causal_attention(ref.query_conv(xr), ref.key_conv(xr))
    ((yr * g.double()).sum() + (ar * ga.double()).sum()).backward()
    rel = lambda a, b: (a.detach().double().cpu() - b).abs().max().item() / max(1.0, b.abs().max().item())
    errs = dict(y=rel(y, yr.detach()), attn=rel(attn, ar.detach()), dx=rel(xd.grad, xr.grad))
    for (n, p), (_, pr) in zip(m.named_parameters(), ref.named_parameters()):
        assert p.grad is not None, n
        errs[n] = rel(p.grad, pr.grad)
    print("ERR", json.dumps(dict(what="module causal", err={n: float(f"{e:.2e}") for n, e in errs.items()})))
    npix = 2 * 4 * 7 * 6
    assert len(errs) == 10 and errs.pop("key_conv.bias") <= 1e-3 * npix ** 0.5, errs
    assert all(e <= 1e-3 for e in errs.values()), errs


def test_torch_compile_fullgraph():
    import ccnet_b200  # noqa: F401
    q, k, v, _ = (t.cuda() for t in _inputs((1, 16, 64, 3, 8, 9), torch.float32, seed=3))

    def f(q, k, v):
        out, lse = torch.ops.cca.forward3d(q, k, v, True)
        attn = torch.ops.cca.attention3d(q, k, "auto", True)
        so, sl = torch.ops.cca.forward3d_step(q[:, :, 2], k[:, :, 2], v[:, :, 2], k[:, :, :2], v[:, :, :2])
        return out * 2, lse, attn, so, sl

    fc = torch.compile(f, fullgraph=True)
    for a, b in zip(fc(q, k, v), f(q, k, v)):
        assert torch.equal(a, b)
