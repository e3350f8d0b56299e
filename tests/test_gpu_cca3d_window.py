"""GPU tests (H100: ``pytest -m gpu``) of time windows in causal criss-cross attention over clips and of the ring-buffer
step: the windowed forward, backward, map and map backward of both kernel families against the fp64 oracle of
tests/cca3d_window_oracle.py in fp32, bf16 and fp16 at the budgets of the causal tests; W >= T - 1 bit for bit the
unwindowed op; the deterministic mode; a generic clip longer than the unwindowed bound; the ring step frame by frame against
the windowed clip forward; the windowed module; torch.compile.  Each comparison prints one ``ERR {json}`` line (run with
``-s``)."""
import json

import pytest
import torch

import cca3d_window_oracle as OW
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


def _reference(q, k, v, dout, window):
    q, k, v, dout = (t.double() for t in (q, k, v, dout))
    out, lse = OW.cca3d_window_forward(q, k, v, window)
    dq, dk, dv = OW.cca3d_window_backward(dout, q, k, v, window)
    return dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv)


def _run(q, k, v, dout, window, impl="auto", deterministic=None):
    from ccnet_b200 import cca3d_backward, cca3d_forward
    q, k, v, dout = (t.cuda() for t in (q, k, v, dout))
    out, lse = cca3d_forward(q, k, v, impl, deterministic, causal=True, window=window)
    dq, dk, dv = cca3d_backward(dout, q, k, v, out, lse, impl, deterministic, causal=True, window=window)
    torch.cuda.synchronize()
    return dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv)


def _check(got, ref, budget, what):
    errs = tb.check({n: t.cpu() for n, t in got.items()}, ref, budget, what)
    print("ERR", json.dumps(dict(what=what, err={n: float(f"{e:.2e}") for n, e in errs.items()})))
    return errs


# (B, Cq, C, T, H, W): T in {2, 5, 9, 17, 32}, Cq in {16, 48, 64}, one-tile and tiled lines
SHAPES = [
    (2, 48, 128, 2, 9, 8),
    (1, 64, 64, 5, 7, 11),
    (1, 48, 64, 9, 5, 7),
    (1, 16, 64, 17, 5, 4),
    (1, 16, 64, 32, 4, 5),
    (1, 16, 64, 5, 129, 20),
]
SIDS = ["x".join(map(str, s)) for s in SHAPES]
CASES = [(s, w) for s in SHAPES for w in sorted({1, 3, max(1, s[3] - 2)})]
CIDS = [f"{'x'.join(map(str, s))}-W{w}" for s, w in CASES]


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("shape,window", CASES, ids=CIDS)
def test_windowed_forward_backward_vs_oracle(shape, window, dtype):
    budget = dict(BUDGETS[dtype])
    if dtype == torch.float16 and max(shape[4:]) > 112:
        budget["lse"] = tb.FP32_BUDGET["lse"]
    q, k, v, dout = _inputs(shape, dtype, seed=sum(shape) + window)
    ref = _reference(q, k, v, dout, window)
    _check(_run(q, k, v, dout, window), ref, budget, f"tc {shape} W={window} {dtype}")
    _check(_run(q, k, v, dout, window, impl="simt"), ref, SIMT_BUDGETS[dtype], f"simt {shape} W={window} {dtype}")


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("shape", [SHAPES[2], SHAPES[4], SHAPES[5]], ids=[SIDS[2], SIDS[4], SIDS[5]])
def test_windowed_map_and_its_backward_vs_oracle(shape, dtype):
    """the map (time entries outside [t - W, t) exactly 0) and dq, dk of both families at W = 3"""
    from ccnet_b200.functional import cca3d_attention_backward, cca3d_attention_forward
    B, Cq, C, T, H, W = shape
    window = 3
    q, k, _, _ = _inputs(shape, dtype, seed=sum(shape) + 3)
    g = torch.Generator().manual_seed(5)
    dattn = torch.randn(B, T, H, W, H + W + T, generator=g)
    a_ref = OW.cca3d_window_attention(q.double(), k.double(), window)
    dq_ref, dk_ref = OW.cca3d_window_attention_backward(dattn.double(), q.double(), k.double(), window)
    mask = OW.time_mask(T, window=window).view(1, T, 1, 1, T).expand(B, T, H, W, T)
    for impl, budgets in (("auto", BUDGETS), ("simt", SIMT_BUDGETS)):
        qc, kc = q.cuda(), k.cuda()
        attn = cca3d_attention_forward(qc, kc, impl, causal=True, window=window)
        dq, dk = cca3d_attention_backward(dattn.cuda(), attn, qc, kc, impl, causal=True, window=window)
        assert (attn[..., H + W:].cpu()[mask] == 0).all()
        errs = dict(attn=tb.error("out", attn.cpu(), a_ref), dq=tb.error("dq", dq.cpu(), dq_ref), dk=tb.error("dk", dk.cpu(), dk_ref))
        print("ERR", json.dumps(dict(what=f"map {impl} {shape} W={window} {dtype}", err=errs)))
        b = budgets[dtype]
        assert errs["attn"] <= max(b["out"], 1e-2 if dtype != torch.float32 else 0) and errs["dq"] <= b["dq"] and errs["dk"] <= b["dk"], errs


@pytest.mark.parametrize("impl", ["auto", "simt"])
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_window_of_t_minus_1_or_more_is_bitwise_the_causal_op(dtype, impl):
    """one-tile lines, and tiled lines in the deterministic mode (without it the tensor-core 2D passes add their partial
    results in no fixed order, so two calls of the same op differ there)"""
    from ccnet_b200.functional import cca3d_attention_backward, cca3d_attention_forward
    for shape in (SHAPES[2], SHAPES[5]):
        T, det = shape[3], max(shape[4:]) > 112
        q, k, v, dout = (t.cuda() for t in _inputs(shape, dtype, seed=21))
        ref = _run(q, k, v, dout, None, impl, det)
        a0 = cca3d_attention_forward(q, k, impl, det, causal=True)
        da = torch.randn_like(a0)
        g0 = cca3d_attention_backward(da, a0, q, k, impl, det, causal=True)
        for window in (T - 1, T, 4 * T):
            got = _run(q, k, v, dout, window, impl, det)
            assert all(torch.equal(got[n], ref[n]) for n in ref), (shape, window, [n for n in ref if not torch.equal(got[n], ref[n])])
            a = cca3d_attention_forward(q, k, impl, det, causal=True, window=window)
            g = cca3d_attention_backward(da, a, q, k, impl, det, causal=True, window=window)
            assert torch.equal(a, a0) and torch.equal(g[0], g0[0]) and torch.equal(g[1], g0[1]), (shape, window)


def test_deterministic_mode_is_bit_reproducible_on_tiled_lines():
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        shape = (2, 16, 64, 6, 130, 113)
        q, k, v, dout = _inputs(shape, torch.float32, seed=5)
        a, b = _run(q, k, v, dout, 2), _run(q, k, v, dout, 2)
        assert all(torch.equal(a[n], b[n]) for n in a), [n for n in a if not torch.equal(a[n], b[n])]
        _check(a, _reference(q, k, v, dout, 2), tb.FP32_BUDGET, f"deterministic {shape} W=2")
    finally:
        torch.use_deterministic_algorithms(was)


def test_generic_windowed_clip_past_the_unwindowed_key_bound():
    """T = 2100 at 2 x 3 pixels: H + W + T - 2 = 2103 keys is beyond the generic kernels without a window, and 4 + 16 with
    W = 16; forward, backward and the map against the oracle"""
    from ccnet_b200 import cca3d_forward
    from ccnet_b200.functional import cca3d_attention_backward, cca3d_attention_forward
    shape = (1, 8, 16, 2100, 2, 3)
    q, k, v, dout = _inputs(shape, torch.float32, seed=2100)
    with pytest.raises(RuntimeError, match="unsupported shape"):
        cca3d_forward(q.cuda(), k.cuda(), v.cuda(), causal=True)
    got = _run(q, k, v, dout, 16)
    assert got["out"].is_contiguous()
    _check(got, _reference(q, k, v, dout, 16), tb.FP32_SIMT, "simt T=2100 W=16")
    attn = cca3d_attention_forward(q.cuda(), k.cuda(), causal=True, window=16)
    a_ref = OW.cca3d_window_attention(q.double(), k.double(), 16)
    dattn = torch.randn(*attn.shape, generator=torch.Generator().manual_seed(1))
    dq, dk = cca3d_attention_backward(dattn.cuda(), attn, q.cuda(), k.cuda(), causal=True, window=16)
    dq_ref, dk_ref = OW.cca3d_window_attention_backward(dattn.double(), q.double(), k.double(), 16)
    errs = dict(attn=tb.error("out", attn.cpu(), a_ref), dq=tb.error("dq", dq.cpu(), dq_ref), dk=tb.error("dk", dk.cpu(), dk_ref))
    print("ERR", json.dumps(dict(what="map simt T=2100 W=16", err=errs)))
    b = tb.FP32_SIMT
    assert errs["attn"] <= b["out"] and errs["dq"] <= b["dq"] and errs["dk"] <= b["dk"], errs


# ---------------------------------------------------------------------------------------------------------------------
# the ring step
# ---------------------------------------------------------------------------------------------------------------------
def _ring_vs_clip(shape, window, impl, bitwise, deterministic=None, N=None, head0=0):
    """stream the clip through rings of N >= window slots (the oldest frame's slot overwritten once `window` frames are
    held; the first frame goes to slot head0): frame t against frame t of the windowed clip forward"""
    from ccnet_b200 import cca3d_forward, cca3d_step
    q, k, v, _ = (t.cuda() for t in _inputs(shape, torch.float32, seed=sum(shape) + window))
    B, Cq, C, T, H, W = shape
    N = N or window
    out, lse = cca3d_forward(q, k, v, impl, deterministic, causal=True, window=window)
    ref = OW.cca3d_window_forward(q.double().cpu(), k.double().cpu(), v.double().cpu(), window)
    fmt = torch.channels_last_3d if impl == "tc" else torch.contiguous_format
    kr = torch.full((B, Cq, N, H, W), float("nan"), device="cuda").contiguous(memory_format=fmt)
    vr = torch.full((B, C, N, H, W), float("nan"), device="cuda").contiguous(memory_format=fmt)
    S, head = 0, head0
    for t in range(T):
        so, sl = cca3d_step(q[:, :, t], k[:, :, t], v[:, :, t], kr, vr, impl, deterministic, frames=S, head=head)
        if bitwise:
            assert torch.equal(so, out[:, :, t]) and torch.equal(sl, lse[:, t]), (shape, window, t)
        err = tb.error("out", so.cpu(), ref[0][:, :, t])
        assert err <= (tb.FP32_BUDGET if impl == "tc" else tb.FP32_SIMT)["out"], (shape, t, err)
        slot = (head + S) % N
        kr[:, :, slot], vr[:, :, slot] = k[:, :, t], v[:, :, t]
        S, head = (S + 1, head) if S < window else (S, (head + 1) % N)
    print("ERR", json.dumps(dict(what=f"ring {impl} {shape} W={window} N={N}", err=err)))


@pytest.mark.parametrize("window", [1, 3, 7])
def test_ring_step_is_bitwise_the_windowed_clip_forward_on_one_tile_lines(window):
    _ring_vs_clip((2, 16, 64, 2 * window + 5, 9, 8), window, "tc", bitwise=True)


def test_ring_step_deterministic_on_tiled_lines():
    _ring_vs_clip((1, 16, 64, 9, 20, 130), 3, "tc", bitwise=True, deterministic=True)


@pytest.mark.parametrize("window", [1, 4])
def test_generic_ring_step_is_bitwise_the_generic_windowed_clip(window):
    _ring_vs_clip((1, 8, 24, 2 * window + 5, 6, 7), window, "simt", bitwise=True)


@pytest.mark.parametrize("impl", ["tc", "simt"])
def test_ring_step_with_spare_slots_and_a_head(impl):
    _ring_vs_clip((1, 16, 64, 11, 6, 7), 3, impl, bitwise=True, N=5, head0=4)


# ---------------------------------------------------------------------------------------------------------------------
# the module
# ---------------------------------------------------------------------------------------------------------------------
def _windowed_module(C, window, gamma=0.7, seed=0):
    from ccnet_b200 import CrissCrossAttention3D
    torch.manual_seed(seed)
    m = CrissCrossAttention3D(C, causal=True, window=window).cuda()
    with torch.no_grad():
        m.gamma.fill_(gamma)
    return m


@pytest.mark.parametrize("C", [128, 64], ids=["tc", "generic"])
def test_module_ring_step_loop_equals_the_windowed_forward(C):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    m = _windowed_module(C, 3)
    x = torch.randn(2, C, 10, 9, 8, device="cuda")
    with torch.no_grad():
        y = m(x)
        state, ys, ptrs = None, [], set()
        for t in range(10):
            yt, state = m.step(x[:, :, t], state)
            ys.append(yt)
            ptrs.add((state.k.data_ptr(), state.v.data_ptr()))
            assert state.frames == min(t + 1, 3) and state.k.shape[2] == 3
        err = (torch.stack(ys, 2) - y).abs().max().item()
    print("ERR", json.dumps(dict(what=f"module ring step C={C}", err=err)))
    assert len(ptrs) == 1 and err <= 1e-4, (ptrs, err)


def test_windowed_module_vs_oracle_with_gradients():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    m = _windowed_module(128, 2)
    ref = OW.WindowCrissCrossAttention3DOracle(128, window=2).double()
    ref.load_state_dict({n: p.detach().double().cpu() for n, p in m.state_dict().items()})
    x = torch.randn(2, 128, 6, 7, 6)
    xd = x.cuda().requires_grad_(True)
    y, attn = m(xd, return_attention=True)
    g = torch.randn_like(x)
    ga = torch.randn(*attn.shape)
    ((y * g.cuda()).sum() + (attn * ga.cuda()).sum()).backward()
    xr = x.double().requires_grad_(True)
    yr = ref(xr)
    ar = OW.cca3d_window_attention(ref.query_conv(xr), ref.key_conv(xr), 2)
    ((yr * g.double()).sum() + (ar * ga.double()).sum()).backward()
    rel = lambda a, b: (a.detach().double().cpu() - b).abs().max().item() / max(1.0, b.abs().max().item())
    errs = dict(y=rel(y, yr.detach()), attn=rel(attn, ar.detach()), dx=rel(xd.grad, xr.grad))
    for (n, p), (_, pr) in zip(m.named_parameters(), ref.named_parameters()):
        assert p.grad is not None, n
        errs[n] = rel(p.grad, pr.grad)
    print("ERR", json.dumps(dict(what="module windowed", err={n: float(f"{e:.2e}") for n, e in errs.items()})))
    npix = 2 * 6 * 7 * 6
    assert len(errs) == 10 and errs.pop("key_conv.bias") <= 1e-3 * npix ** 0.5, errs
    assert all(e <= 1e-3 for e in errs.values()), errs


def test_torch_compile_fullgraph_over_the_window_and_ring_arguments():
    import ccnet_b200  # noqa: F401
    q, k, v, _ = (t.cuda() for t in _inputs((1, 16, 64, 5, 8, 9), torch.float32, seed=3))
    kr, vr = (t.contiguous(memory_format=torch.channels_last_3d) for t in (k, v))

    def f(q, k, v):
        out, lse = torch.ops.cca.forward3d(q, k, v, True, 2)
        attn = torch.ops.cca.attention3d(q, k, "auto", True, 2)
        so, sl = torch.ops.cca.forward3d_step(q[:, :, 4], k[:, :, 4], v[:, :, 4], kr, vr, 2, 2)
        return out * 2, lse, attn, so, sl

    fc = torch.compile(f, fullgraph=True)
    for a, b in zip(fc(q, k, v), f(q, k, v)):
        assert torch.equal(a, b)
    # slots 2, 3 hold frames 2, 3: the step is frame 4 of the clip with window 2
    out, lse = torch.ops.cca.forward3d(q, k, v, True, 2)
    so, sl = f(q, k, v)[3:]
    assert torch.equal(so, out[:, :, 4]) and torch.equal(sl, lse[:, 4])
