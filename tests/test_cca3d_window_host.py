"""CPU tests of time windows in causal criss-cross attention over clips and of the ring-buffer step: the windowed fp64
oracle (tests/cca3d_window_oracle.py) against a per-pixel loop and the unwindowed oracle; the ring step
oracle; the C entry points' symbols, argument types and validation; the plans of windowed calls and ring steps; the fake
implementations; and the module's construction errors."""
import os

import pytest
import torch

import cca3d_causal_oracle as OC
import cca3d_window_oracle as OW
from ccnet_b200 import build, capi


def _qkv(B, Cq, C, T, H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    mk = lambda c: torch.randn(B, c, T, H, W, generator=g, dtype=torch.float64)
    return mk(Cq), mk(Cq), mk(C)


SHAPES = [(1, 2, 3, 6, 3, 4), (2, 3, 2, 5, 2, 3), (1, 2, 3, 9, 1, 2)]


def _bruteforce(q, k, v, window):
    """one pixel at a time: its column (self masked), its row and the frames t - window <= s < t, one softmax"""
    B, _, T, H, W = q.shape
    out, lse = torch.zeros_like(v), torch.zeros(B, T, H, W, dtype=q.dtype)
    for b in range(B):
        for t in range(T):
            for h in range(H):
                for w in range(W):
                    keys = [(t, g, w) for g in range(H) if g != h] + [(t, h, g) for g in range(W)]
                    keys += [(s, h, w) for s in range(max(0, t - window), t)]
                    e = torch.stack([(q[b, :, t, h, w] * k[b, :, s, g, x]).sum() for s, g, x in keys])
                    a = torch.softmax(e, 0)
                    lse[b, t, h, w] = torch.logsumexp(e, 0)
                    out[b, :, t, h, w] = sum(a[i] * v[b, :, s, g, x] for i, (s, g, x) in enumerate(keys))
    return out, lse


@pytest.mark.parametrize("window", [1, 2, 4])
@pytest.mark.parametrize("shape", SHAPES[:2])
def test_windowed_oracle_matches_a_per_pixel_loop(shape, window):
    q, k, v = _qkv(*shape, seed=window)
    for a, b in zip(OW.cca3d_window_forward(q, k, v, window), _bruteforce(q, k, v, window)):
        assert (a - b).abs().max().item() < 1e-12


@pytest.mark.parametrize("window", [1, 3])
@pytest.mark.parametrize("shape", SHAPES)
def test_windowed_logits_are_the_causal_logits_with_older_time_keys_masked(shape, window):
    q, k, _ = _qkv(*shape, seed=2)
    B, Cq, C, T, H, W = shape
    e, ew = OC.cca3d_causal_logits(q, k), OW.cca3d_window_logits(q, k, window)
    old = torch.ones(T, T, dtype=torch.bool).tril(-window - 1).view(1, T, 1, 1, T)
    assert torch.equal(ew[..., :H + W], e[..., :H + W]) and torch.equal(ew[..., H + W:], e[..., H + W:].masked_fill(old, float("-inf")))


@pytest.mark.parametrize("shape", SHAPES)
def test_window_of_t_minus_1_or_more_is_the_causal_oracle_and_masked_entries_are_0(shape):
    q, k, v = _qkv(*shape, seed=1)
    B, Cq, C, T, H, W = shape
    dout = torch.randn_like(v)
    ref = OC.cca3d_causal_forward(q, k, v) + OC.cca3d_causal_backward(dout, q, k, v)
    for window in (None, T - 1, T, T + 5):
        got = OW.cca3d_window_forward(q, k, v, window) + OW.cca3d_window_backward(dout, q, k, v, window)
        assert all(torch.equal(a, b) for a, b in zip(got, ref)), window
    for window in (1, 2):
        a = OW.cca3d_window_attention(q, k, window)
        t, s = torch.arange(T).view(T, 1), torch.arange(T).view(1, T)
        outside = ((s >= t) | (s < t - window)).view(1, T, 1, 1, T).expand(B, T, H, W, T)
        assert torch.equal(OW.time_mask(T, window=window), (s >= t) | (s < t - window))
        assert (a[..., H + W:][outside] == 0).all() and (a[..., H + W:][~outside] > 0).all()
        assert (a.sum(-1) - 1).abs().max().item() < 1e-12


@pytest.mark.parametrize("window", [1, 3])
@pytest.mark.parametrize("shape", SHAPES)
def test_windowed_closed_form_gradients_match_autograd(shape, window):
    q, k, v = _qkv(*shape, seed=3)
    dout, dattn = torch.randn_like(v), torch.randn(*OC.cca3d_causal_logits(q, k).shape, dtype=torch.float64)
    qa, ka, va = (t.clone().requires_grad_(True) for t in (q, k, v))
    out, _ = OW.cca3d_window_forward(qa, ka, va, window)
    ref = torch.autograd.grad(out, (qa, ka, va), dout)
    for a, b in zip(OW.cca3d_window_backward(dout, q, k, v, window), ref):
        assert (a - b).abs().max().item() < 1e-10
    attn = OW.cca3d_window_attention(qa, ka, window)
    ref = torch.autograd.grad(attn, (qa, ka), dattn)
    for a, b in zip(OW.cca3d_window_attention_backward(dattn, q, k, window), ref):
        assert (a - b).abs().max().item() < 1e-10


@pytest.mark.parametrize("window", [1, 3])
def test_ring_step_oracle_streams_the_windowed_clip_oracle(window):
    """a ring of `window` slots written frame by frame (the oldest slot overwritten once full) over T > 2 window + 1 frames,
    so that it wraps more than once: frame t stepped with the last min(t, window) frames is frame t of the windowed clip"""
    T = 2 * window + 4
    q, k, v = _qkv(2, 3, 4, T, 3, 2, seed=7 + window)
    out, lse = OW.cca3d_window_forward(q, k, v, window)
    kr, vr = torch.zeros(2, 3, window, 3, 2, dtype=q.dtype), torch.zeros(2, 4, window, 3, 2, dtype=q.dtype)
    S = head = 0
    for t in range(T):
        so, sl = OW.cca3d_step_ring(q[:, :, t], k[:, :, t], v[:, :, t], kr, vr, S, head)
        assert (so - out[:, :, t]).abs().max().item() < 1e-12 and (sl - lse[:, t]).abs().max().item() < 1e-12, t
        slot = (head + S) % window
        kr[:, :, slot], vr[:, :, slot] = k[:, :, t], v[:, :, t]
        S, head = (S + 1, head) if S < window else (S, (head + 1) % window)
    assert head != 0 or T % window == 0


def test_ring_step_oracle_with_spare_slots_and_head():
    q, k, v = _qkv(1, 2, 3, 4, 2, 3, seed=11)
    N, head = 6, 4                                          # frames 0, 1, 2 in slots 4, 5, 0
    kr, vr = torch.randn(1, 2, N, 2, 3, dtype=q.dtype), torch.randn(1, 3, N, 2, 3, dtype=q.dtype)
    for j, slot in enumerate((4, 5, 0)):
        kr[:, :, slot], vr[:, :, slot] = k[:, :, j], v[:, :, j]
    so, sl = OW.cca3d_step_ring(q[:, :, 3], k[:, :, 3], v[:, :, 3], kr, vr, 3, head)
    out, lse = OC.cca3d_causal_forward(q, k, v)
    assert (so - out[:, :, 3]).abs().max().item() < 1e-12 and (sl - lse[:, 3]).abs().max().item() < 1e-12


NEW = {"cca_b200_forward3d_window": "cca_b200_forward3d", "cca_b200_backward3d_window": "cca_b200_backward3d",
       "cca_b200_attention_forward3d_window": "cca_b200_attention_forward3d",
       "cca_b200_attention_backward3d_window": "cca_b200_attention_backward3d"}


def test_new_symbols_and_argtypes():
    lib = capi.load()
    hdr = open(os.path.join(build.HERE, "..", "include", "cca_b200.h")).read()
    for name, base in NEW.items():
        assert name in hdr and getattr(lib, name) is not None
        res, args = capi.SYMBOLS[name]
        bres, bargs = capi.SYMBOLS[base]
        # the existing entry point with an int window before dtype
        assert res == bres and args == bargs[:-3] + [bargs[-3]] + bargs[-3:], name
    res, args = capi.SYMBOLS["cca_b200_forward3d_step_ring"]
    bres, bargs = capi.SYMBOLS["cca_b200_forward3d_step"]
    assert "cca_b200_forward3d_step_ring" in hdr and res == bres and len(args) == len(bargs) + 2
    assert lib.cca_b200_version() == 200


def test_window_calls_reject_bad_arguments_before_any_cuda_call():
    lib = capi.load()
    err = lib.cca_b200_last_error
    p, causal = 16, capi.CCA_FLAG_CAUSAL
    for window, flags, what in ((-1, causal, b"negative"), (3, 0, b"CAUSAL"), (3, capi.CCA_FLAG_NHWC, b"CAUSAL")):
        assert lib.cca_b200_forward3d_window(*(p,) * 6, 1 << 30, 1, 8, 16, 5, 4, 4, window, capi.CCA_F32, flags, None) == -1
        assert what in err()
        assert lib.cca_b200_backward3d_window(*(p,) * 10, 1 << 30, 1, 8, 16, 5, 4, 4, window, capi.CCA_F32, flags, None) == -1
        assert what in err()
        assert lib.cca_b200_attention_forward3d_window(*(p,) * 4, 1 << 30, 1, 8, 5, 4, 4, window, capi.CCA_F32, flags, None) == -1
        assert what in err()
        assert lib.cca_b200_attention_backward3d_window(*(p,) * 7, 1 << 30, 1, 8, 5, 4, 4, window, capi.CCA_F32, flags,
                                                        None) == -1
        assert what in err()
    # a valid window passes its check and stops at the workspace check, before anything touches a device
    assert lib.cca_b200_forward3d_window(*(p,) * 6, 16, 1, 8, 16, 5, 4, 4, 2, capi.CCA_F32, causal, None) == -3


def test_ring_step_rejects_bad_arguments_before_any_cuda_call():
    lib = capi.load()
    err = lib.cca_b200_last_error
    p, nhwc = 16, capi.CCA_FLAG_NHWC

    def call(N=4, S=3, head=0, ptrs=(p,) * 8, nbytes=1 << 30):
        return lib.cca_b200_forward3d_step_ring(*ptrs, nbytes, 1, 16, 64, N, S, head, 5, 5, capi.CCA_F32, nhwc, None)
    assert call(S=-1) == -1 and b"negative" in err()
    assert call(N=2, S=3) == -1 and b"slots" in err()
    assert call(head=4) == -1 and b"head" in err()
    assert call(head=-1) == -1 and b"head" in err()
    for i in (3, 4):
        ptrs = [p] * 8
        ptrs[i] = None
        assert call(ptrs=tuple(ptrs)) == -1 and b"null" in err(), i
        assert call(S=0, ptrs=tuple(ptrs), nbytes=16) == -3        # no frame is read: NULL rings pass
    assert call(N=0, S=0, head=5, nbytes=16) == -3                 # (head is not read without slots)
    assert call(nbytes=16) == -3 and b"workspace" in err()


def _record_plans(monkeypatch, fn):
    """run fn under FakeTensorMode with _plan stopping every call: the coverage queries the plans asked, then answered"""
    import ccnet_b200.functional as F_
    from torch._subclasses.fake_tensor import FakeTensorMode
    asked, flags = [], []

    def plan(impl, det, covered, q, v=None, causal=False):
        asked.append(covered)
        raise RuntimeError("stop at the plan")
    monkeypatch.setattr(F_, "_plan", plan)
    with FakeTensorMode():
        fn(F_)
    lib = capi.load()
    calls = []
    real = lib.cca_b200_tc3d_supported
    monkeypatch.setattr(lib, "cca_b200_tc3d_supported", lambda *a: calls.append(a) or real(*a), raising=False)
    answers = [covered() for covered in asked]
    return calls, answers


def test_windowed_calls_plan_by_the_clip_coverage(monkeypatch):
    """a window does not change which family runs: T <= 32 on the tensor cores, longer windowed clips on the generic kernels"""
    def fn(F_):
        for T in (9, 32, 33, 2100):
            q, v = torch.empty(1, 16, T, 2, 3, device="cuda"), torch.empty(1, 64, T, 2, 3, device="cuda")
            with pytest.raises(RuntimeError, match="stop at the plan"):
                F_.cca3d_forward(q, q, v, causal=True, window=4)
    calls, answers = _record_plans(monkeypatch, fn)
    assert [c[4] for c in calls] == [9, 32, 33, 2100] and answers[2:] == [False, False]


def test_ring_steps_plan_by_the_frames_they_read(monkeypatch):
    def fn(F_):
        q, v = torch.empty(1, 16, 9, 9, device="cuda"), torch.empty(1, 64, 9, 9, device="cuda")
        kc, vc = torch.empty(1, 16, 40, 9, 9, device="cuda"), torch.empty(1, 64, 40, 9, 9, device="cuda")
        for frames in (None, 0, 31, 32):
            with pytest.raises(RuntimeError, match="stop at the plan"):
                F_.cca3d_step(q, q, v, kc, vc, frames=frames, head=7)
    calls, answers = _record_plans(monkeypatch, fn)
    assert [c[4] for c in calls] == [41, 1, 32, 33] and answers[0] is False and answers[3] is False


def test_python_layer_rejects_bad_windows_and_ring_indices():
    import ccnet_b200.functional as F_
    assert F_._time_window(False, None) == 0 and F_._time_window(True, None) == 0 and F_._time_window(True, 3) == 3
    for causal, window in ((False, 3), (True, 0), (True, -2), (True, 2.5), (True, True)):
        with pytest.raises(ValueError):
            F_._time_window(causal, window)
    for frames, head in ((5, 0), (-1, 0), (2, 4), (2, -1)):
        with pytest.raises(ValueError, match="frames"):
            _step_args(F_, frames, head)


def _step_args(F_, frames, head):
    from torch._subclasses.fake_tensor import FakeTensorMode
    with FakeTensorMode():
        q = torch.empty(1, 2, 3, 3, device="cuda")
        F_.cca3d_step(q, q, q, torch.empty(1, 2, 4, 3, 3, device="cuda"), torch.empty(1, 2, 4, 3, 3, device="cuda"),
                      frames=frames, head=head)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("T", [5, 40])
def test_fake_implementations_of_the_window_and_ring_arguments(dtype, T):
    import ccnet_b200  # noqa: F401
    from ccnet_b200.functional import tc3d_eligible
    from torch._subclasses.fake_tensor import FakeTensorMode
    fmt = torch.channels_last_3d if tc3d_eligible(2, 16, 64, T, 20, 30, dtype) else torch.contiguous_format
    with FakeTensorMode():
        q = torch.empty(2, 16, T, 20, 30, device="cuda", dtype=dtype)
        v = torch.empty(2, 64, T, 20, 30, device="cuda", dtype=dtype)
        out, lse = torch.ops.cca.forward3d(q, q, v, True, 3)
        assert out.shape == v.shape and out.is_contiguous(memory_format=fmt) and lse.shape == (2, T, 20, 30)
        grads = torch.ops.cca.backward3d(out, q, q, v, out, lse, True, 3)
        assert all(g.is_contiguous(memory_format=fmt) for g in grads)
        attn = torch.ops.cca.attention3d(q, q, "auto", True, 3)
        assert attn.shape == (2, T, 20, 30, 50 + T) and attn.dtype == torch.float32
        assert [g.shape for g in torch.ops.cca.attention3d_backward(attn, attn, q, q, "auto", True, 3)] == [q.shape] * 2
        with pytest.raises(ValueError):
            torch.ops.cca.forward3d(q, q, v, False, 3)
        # a ring of T slots, 4 of them filled: the step plans for a clip of 5 frames
        o, l = torch.ops.cca.forward3d_step(q[:, :, 0], q[:, :, 0], v[:, :, 0], q, v, 4, 1)
        fmt2 = torch.channels_last if tc3d_eligible(2, 16, 64, 5, 20, 30, dtype) else torch.contiguous_format
        assert o.shape == v[:, :, 0].shape and o.is_contiguous(memory_format=fmt2) and l.shape == (2, 20, 30)


def test_windowed_module_construction():
    from ccnet_b200 import CrissCrossAttention3D, RingState
    m = CrissCrossAttention3D(64, causal=True, window=5)
    assert m.window == 5 and CrissCrossAttention3D(64, causal=True).window is None
    assert list(m.state_dict()) == list(CrissCrossAttention3D(64).state_dict())
    for kw in (dict(window=3), dict(causal=True, window=0), dict(causal=True, window=-1), dict(causal=True, window=1.5)):
        with pytest.raises(ValueError):
            CrissCrossAttention3D(64, **kw)
    assert RingState._fields == ("k", "v", "frames", "head")
    with pytest.raises(ValueError, match="max_frames"):
        m.step(torch.randn(1, 64, 3, 3, device="meta"), max_frames=4)
