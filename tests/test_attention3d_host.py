"""CPU tests of the attention map of criss-cross attention over clips: the fp64 oracle (tests/attn3d_budget.py) against the
reference's own maps and gradients through T = 1, fp64 autograd and the 3D op's output; the emulated kernels inside their
budget and a dropped MMA outside it; the fp16 rounding chain; argument validation and workspace sizes of the C entry
points; the fake implementations of torch.ops.cca.attention3d; and the new kernels' resources."""
import glob
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import attn3d_budget as A3
import cca3d_oracle as O3
from ccnet_b200 import build, capi

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "attn_*.npz")))


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p) for p in FIXTURES])
def test_t1_map_and_gradients_reproduce_the_reference_fixtures(path):
    """T = 1: the 3D oracle module (the fixture's parameters as 1x1x1 convs) gives the reference's maps as attn[..., :H+W],
    a time entry of exactly 0, and the reference's gradients of a loss on the maps"""
    f = np.load(path)
    C = f["x"].shape[1]
    m = O3.CrissCrossAttention3DOracle(C).double()
    m.load_state_dict(O3.conv3d_state({n[2:]: torch.from_numpy(f[n]).double() for n in f.files if n.startswith("p_")}))
    x = torch.from_numpy(f["x"]).double().unsqueeze(2).requires_grad_(True)
    H, W = x.shape[3], x.shape[4]
    y, loss = x, 0
    for i in range(int(f["R"])):
        a = A3.attention_map3d(m.query_conv(y), m.key_conv(y))
        assert a.shape == (x.shape[0], 1, H, W, H + W + 1) and a[..., H + W].abs().max().item() == 0
        assert (a[:, 0, ..., :H + W] - torch.from_numpy(f[f"A_{i}"]).double()).abs().max().item() < 1e-6
        loss = loss + (a[:, 0, ..., :H + W] * torch.from_numpy(f[f"R_{i}"]).double()).sum()
        y = m(y)
    loss.backward()
    tol = lambda r: 1e-5 * max(1.0, np.abs(r).max())
    assert np.abs(x.grad.squeeze(2).numpy() - f["dx"]).max() < tol(f["dx"])
    for n, p in m.named_parameters():
        g = p.grad.reshape(f["d_" + n].shape).numpy() if p.grad is not None else np.zeros(f["d_" + n].shape)
        assert np.abs(g - f["d_" + n]).max() < tol(f["d_" + n]), n


@pytest.mark.parametrize("shape", [(2, 8, 3, 5, 6), (1, 4, 1, 4, 7), (1, 4, 5, 1, 11), (1, 4, 4, 13, 1), (2, 16, 6, 9, 7)])
def test_closed_form_backward_matches_fp64_autograd(shape):
    g = torch.Generator().manual_seed(1)
    q, k = (torch.randn(shape, generator=g, dtype=torch.float64).requires_grad_(True) for _ in range(2))
    _, _, T, H, W = shape
    a = A3.attention_map3d(q, k)
    assert a[..., :H].diagonal(dim1=2, dim2=4).abs().max() == 0                  # column self entries exactly 0
    assert a[..., H + W:].diagonal(dim1=1, dim2=4).abs().max() == 0              # time self entries exactly 0
    assert torch.allclose(a.sum(-1), torch.ones_like(a.sum(-1)))
    r = torch.randn(a.shape, generator=g, dtype=torch.float64)
    gq, gk = torch.autograd.grad((a * r).sum(), (q, k))
    dq, dk = A3.attention_map3d_backward(r, q.detach(), k.detach())
    assert torch.allclose(dq, gq, atol=1e-12) and torch.allclose(dk, gk, atol=1e-12)


@pytest.mark.parametrize("shape", [(2, 8, 16, 3, 5, 6), (1, 4, 8, 1, 4, 7), (1, 4, 8, 5, 1, 3)])
def test_map_times_v_is_the_3d_forward_output(shape):
    B, Cq, C, T, H, W = shape
    g = torch.Generator().manual_seed(2)
    q, k = (torch.randn(B, Cq, T, H, W, generator=g, dtype=torch.float64) for _ in range(2))
    v = torch.randn(B, C, T, H, W, generator=g, dtype=torch.float64)
    ah, aw, at = A3._parts(A3.attention_map3d(q, k), H, W)
    o = (torch.einsum("bthwg,bctgw->bcthw", ah, v) + torch.einsum("bthwg,bcthg->bcthw", aw, v)
         + torch.einsum("bthws,bcshw->bcthw", at, v))
    out, _ = O3.cca3d_forward(q, k, v)
    assert (o - out).abs().max().item() < 1e-12


def _native16(dtype, H, W, T):
    from ccnet_b200.functional import _upcast
    return not _upcast(dtype, H, W, False, T)


@pytest.mark.parametrize("T", [1, 4])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["fp32", "bf16", "fp16"])
def test_emulated_kernels_are_inside_their_budget_and_a_dropped_mma_is_not(dtype, T):
    """the emulated kernels sit >= 3x below the budget, a dq item without one of its 16-channel MMAs >= 3x above it"""
    g = torch.Generator().manual_seed(3)
    q, k = ((torch.randn(1, 32, T, 9, 11, generator=g) * 0.7).to(dtype) for _ in range(2))
    da = torch.randn(1, T, 9, 11, 20 + T, generator=g)
    native = _native16(dtype, 9, 11, T)
    ref = A3.reference(q, k, da)
    emu = A3.emulate(q, k, da, dtype, native)
    bud = A3.budget(emu, ref, dtype)
    errs = A3.check(emu, ref, bud)
    assert all(3 * e <= bud[n] for n, e in errs.items()), (errs, bud)
    bad = A3.emulate(q, k, da, dtype, native, drop_kstep=True)
    assert A3.error(bad["dq"], ref["dq"]) >= 3 * bud["dq"]
    with pytest.raises(AssertionError):
        A3.check(bad, ref, bud)


def test_t1_emulation_is_the_2d_emulation():
    """at T = 1 the time pass adds nothing: the emulated map and gradients are those of the 2D map kernels"""
    import attn_budget as AB
    g = torch.Generator().manual_seed(4)
    for dtype in (torch.float32, torch.float16):
        q, k = ((torch.randn(2, 16, 1, 7, 9, generator=g) * 0.7).to(dtype) for _ in range(2))
        da = torch.randn(2, 1, 7, 9, 17, generator=g)
        e3 = A3.emulate(q, k, da, dtype)
        e2 = AB.emulate(q[:, :, 0], k[:, :, 0], da[:, 0, ..., :16], dtype)
        assert torch.equal(e3["attn"][:, 0, ..., :16], e2["attn"]) and e3["attn"][..., 16].abs().max() == 0
        assert torch.equal(e3["dq"][:, :, 0], e2["dq"]) and torch.equal(e3["dk"][:, :, 0], e2["dk"])


def test_fp16_rounding_chain_of_the_native_map_backward():
    """native fp16 dq, dk are rounded three times (column part stored, row part reduce-added, time part added).  With exact
    dS and fp16 inputs that chain alone stays >= 2.5x inside the fp16 op's gradient budget (tests/f16_budget.py), as the
    3D op's does, so fp16 runs natively for T > 1; bf16 with T > 1 runs on the fp32 kernels (functional._upcast)."""
    from f16_budget import F16_BUDGET
    rnd = lambda x: x.half().double()
    worst = {}
    for shape in [(1, 64, 4, 12, 10), (1, 32, 8, 9, 11), (2, 16, 3, 20, 15)]:
        B, Cq, T, H, W = shape
        g = torch.Generator().manual_seed(sum(shape))
        q, k = (rnd(torch.randn(shape, generator=g, dtype=torch.float64) * 0.7) for _ in range(2))
        da = torch.randn(B, T, H, W, H + W + T, generator=g, dtype=torch.float64)
        a = A3.attention_map3d(q, k)
        ds = a * (da - (a * da).sum(-1, keepdim=True))
        for n, (c, r, t) in zip(("dq", "dk"), A3._dqdk(ds, q, k, H, W)):
            ref = c + r + t
            worst[n] = max(worst.get(n, 0.0), (rnd(rnd(rnd(c) + rnd(r)) + t) - ref).abs().max().item() / max(1.0, ref.abs().max().item()))
    print("fp16 three roundings", worst)
    assert all(F16_BUDGET[n] >= 2.5 * e for n, e in worst.items()), worst
    assert _native16(torch.float16, 97, 97, 8) and not _native16(torch.bfloat16, 97, 97, 8) and _native16(torch.bfloat16, 9, 9, 1)


def test_3d_map_symbols_are_exported():
    lib = capi.load()
    for name in ("cca_b200_attention_tc3d_supported", "cca_b200_attention_workspace_bytes3d", "cca_b200_attention_forward3d",
                 "cca_b200_attention_backward3d"):
        assert name in capi.SYMBOLS and getattr(lib, name) is not None
    assert lib.cca_b200_version() == 200                  # an addition to version 0.2.0


def test_3d_map_entry_points_reject_bad_arguments_before_any_cuda_call():
    lib = capi.load()
    err, big, p = lib.cca_b200_last_error, 1 << 30, 16    # p: any non-null address; nothing below touches it
    both = capi.CCA_FLAG_FORCE_SIMT | capi.CCA_FLAG_FORCE_TC
    for fn, n in ((lib.cca_b200_attention_forward3d, 4), (lib.cca_b200_attention_backward3d, 7)):
        def call(ptrs=(p,) * n, nbytes=big, B=1, Cq=16, T=4, H=5, W=5, dtype=capi.CCA_F32, flags=0):
            return fn(*ptrs, nbytes, B, Cq, T, H, W, dtype, flags, None)
        for i in range(n):
            assert call(ptrs=(p,) * i + (None,) + (p,) * (n - 1 - i)) == -1 and b"null" in err()
        assert call(B=0) == -1 and b"dimension" in err()
        assert call(Cq=-16) == -1 and b"dimension" in err()
        for T in (0, -3):
            assert call(T=T) == -1 and b"dimension" in err()
        assert call(B=1 << 16, T=1 << 15) == -2 and b"large" in err()          # B*T past 2^31
        assert call(B=2, T=32, H=1 << 14, W=1 << 14) == -2 and b"large" in err()   # map past 2^40 elements
        assert call(dtype=7) == -1 and b"dtype" in err()
        assert call(flags=both) == -1 and b"exclusive" in err()
        assert call(flags=both | capi.CCA_FLAG_NHWC) == -1 and b"exclusive" in err()
        assert call(nbytes=0) == -3 and b"workspace" in err()
    # attn / dattn need only float alignment: an address that is not one is refused
    assert lib.cca_b200_attention_forward3d(p, p, p + 2, p, big, 1, 16, 4, 5, 5, capi.CCA_F32, 0, None) == -1
    assert b"aligned" in err()
    assert lib.cca_b200_attention_backward3d(p, p + 2, p, p, p, p, p, big, 1, 16, 4, 5, 5, capi.CCA_F32, 0, None) == -1
    assert b"aligned" in err()
    assert lib.cca_b200_attention_backward3d(p + 1, p, p, p, p, p, p, big, 1, 16, 4, 5, 5, capi.CCA_F32, 0, None) == -1


def _a16(x):
    return (x + 15) // 16 * 16


@pytest.mark.parametrize("shape", [(1, 64, 8, 97, 97), (2, 16, 3, 130, 20), (1, 32, 32, 65, 65), (2, 8, 40, 9, 9)])
def test_3d_map_workspace_sizes(shape):
    """one size covers either family: forward the statistics planes of the frames view plus the time plane (the 3D op's
    forward workspace without its counters' role), backward rho of every pixel (+ the dQ, dK planes in deterministic fp32
    mode on tiled lines)"""
    B, Cq, T, H, W = shape
    lib = capi.load()
    npix = B * T * H * W
    nparts = -(-H // 112) + -(-W // 112)
    nhwc, det = capi.CCA_FLAG_NHWC, capi.CCA_FLAG_NHWC | capi.CCA_FLAG_DETERMINISTIC
    fwd = lib.cca_b200_attention_workspace_bytes3d(0, *shape, capi.CCA_F32, nhwc)
    assert fwd == _a16((nparts + 1) * npix * 4) + _a16(B * T * 4)
    assert fwd == lib.cca_b200_workspace_bytes3d(capi.CCA_WS_FORWARD, B, Cq, 64, T, H, W, capi.CCA_F32, nhwc)
    bwd = lib.cca_b200_attention_workspace_bytes3d(1, *shape, capi.CCA_F32, nhwc)
    assert bwd == max((npix * 4 + 255) // 256 * 256, npix * 4 + 16)
    assert bwd == max(lib.cca_b200_attention_workspace_bytes(1, B * T, Cq, H, W, capi.CCA_F32, nhwc), npix * 4 + 16)
    extra = lib.cca_b200_attention_workspace_bytes3d(1, *shape, capi.CCA_F32, det) - bwd
    extra2d = (lib.cca_b200_attention_workspace_bytes(1, B * T, Cq, H, W, capi.CCA_F32, det)
               - lib.cca_b200_attention_workspace_bytes(1, B * T, Cq, H, W, capi.CCA_F32, nhwc))
    assert extra == (extra2d if nparts > 2 else 0) and (nparts == 2 or extra >= 2 * nparts * npix * Cq * 4)
    assert lib.cca_b200_attention_workspace_bytes3d(1, *shape, capi.CCA_BF16, det) == bwd
    assert lib.cca_b200_attention_workspace_bytes3d(0, B, Cq, 0, H, W, capi.CCA_F32, 0) == 0


def test_3d_map_coverage_without_gpu():
    lib = capi.load()
    for T in (0, 33, 64):
        assert lib.cca_b200_attention_tc3d_supported(1, 64, T, 9, 9, capi.CCA_F32) == 0
    assert lib.cca_b200_attention_tc3d_supported(1, 8, 4, 9, 9, capi.CCA_F32) == 0       # Cq = 8
    assert lib.cca_b200_attention_tc3d_supported(1, 64, 4, 897, 9, capi.CCA_F32) == 0    # line > 896
    assert lib.cca_b200_attention_tc3d_supported(1, 64, 4, 9, 9, 7) == 0


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("Cq", [64, 8])
def test_fake_implementations_give_shapes_and_memory_formats(dtype, Cq):
    import ccnet_b200  # noqa: F401  (registers torch.ops.cca)
    from ccnet_b200.functional import attention3d_tc_eligible
    from torch._subclasses.fake_tensor import FakeTensorMode
    cl = attention3d_tc_eligible(2, Cq, 5, 20, 30, dtype)
    if Cq == 8:
        assert not cl
    fmt = torch.channels_last_3d if cl else torch.contiguous_format
    with FakeTensorMode():
        q = torch.empty(2, Cq, 5, 20, 30, device="cuda", dtype=dtype)
        a = torch.ops.cca.attention3d(q, q)
        assert a.shape == (2, 5, 20, 30, 55) and a.dtype == torch.float32 and a.is_contiguous()
        grads = torch.ops.cca.attention3d_backward(a, a, q, q)
        assert all(g.shape == q.shape and g.dtype == dtype and g.is_contiguous(memory_format=fmt) for g in grads)
        grads = torch.ops.cca.attention3d_backward(a, a, q, q, "simt")
        assert all(g.is_contiguous() for g in grads)


def _ptxas(src, tmp_path):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    out = subprocess.run([nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "k.o")],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    return out.stdout + out.stderr


def _frames(report):
    names, frames = [], []
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            names.append(m.group(1))
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            frames.append((names[-1], int(m.group(1)), int(m.group(2)), int(m.group(3))))
    return names, frames


def test_tensor_core_3d_map_kernels_have_no_spills_no_stack_and_no_serialised_wgmma(tmp_path):
    report = _ptxas(os.path.join(build.CSRC, "cca_tc_attn3d.cu"), tmp_path)
    assert "C7514" not in report, [l for l in report.splitlines() if "C7514" in l][:3]
    names, frames = _frames(report)
    # map forward <80, 112> x <fp32, bf16, f16>; backward the same + the fp32 planes mode; time map forward and backward
    # x {T <= 8, 16, 32} x {fp32, bf16, f16}
    assert len([n for n in names if "attn3d_fwd" in n]) == 6 and len([n for n in names if "attn3d_bwd" in n]) == 8, names
    assert len([n for n in names if "cca_time_map_" in n]) == 18, names
    assert len(names) == 32 and len(frames) == 32 and all(f[1:] == (0, 0, 0) for f in frames), frames


def test_generic_3d_map_kernels_have_no_spills_and_no_stack(tmp_path):
    names, frames = _frames(_ptxas(os.path.join(build.CSRC, "cca_simt_attn3d.cu"), tmp_path))
    # map, dq, dk for fp32 / bf16 / f16
    assert len(names) == 9 and len(frames) == 9 and all(f[1:] == (0, 0, 0) for f in frames), frames
