"""CPU tests of criss-cross attention over clips (the 3D op): the fp64 oracle (tests/cca3d_oracle.py) against brute force,
against the reference's own fixtures through T = 1, and against the 2D oracle through H = 1; the C entry points' validation
and workspace sizes; the module's parameters; the fake implementations of torch.ops.cca.forward3d / backward3d; and the
ptxas resources of the time-branch kernels."""
import glob
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import cca3d_oracle as O3
from ccnet_b200 import build, capi
from oracle import cca_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "cca_*.npz")))
T_ = torch.from_numpy


def _qkv(B, Cq, C, T, H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, Cq, T, H, W, generator=g, dtype=torch.float64), torch.randn(B, Cq, T, H, W, generator=g, dtype=torch.float64),
            torch.randn(B, C, T, H, W, generator=g, dtype=torch.float64))


@pytest.mark.parametrize("shape", [(1, 2, 3, 3, 2, 4), (2, 3, 2, 1, 3, 1), (1, 2, 2, 4, 1, 3), (1, 1, 2, 1, 1, 1)])
def test_oracle_matches_brute_force(shape):
    q, k, v = _qkv(*shape)
    out, lse = O3.cca3d_forward(q, k, v)
    ro, rl = O3.cca3d_forward_bruteforce(q, k, v)
    assert (out - ro).abs().max().item() < 1e-12 and (lse - rl).abs().max().item() < 1e-12


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p) for p in FIXTURES])
def test_t1_reproduces_the_reference_fixtures(path):
    """T = 1: the op on the fixture's q, k, v and the module (with the fixture's parameters as 1x1x1 convs, R steps)
    reproduce the reference's outputs and gradients"""
    f = np.load(path)
    q, k, v = (T_(f[n]).double().unsqueeze(2) for n in "qkv")
    out, _ = O3.cca3d_forward(q, k, v)
    assert (out.squeeze(2) - T_(f["o"]).double()).abs().max().item() < 2e-5
    C = f["x"].shape[1]
    m = O3.CrissCrossAttention3DOracle(C)
    m.load_state_dict(O3.conv3d_state({n[2:]: T_(f[n]) for n in f.files if n.startswith("p_")}))
    x = T_(f["x"]).unsqueeze(2).requires_grad_(True)
    y = x
    for _ in range(int(f["R"])):
        y = m(y)
    (y * T_(f["g"]).unsqueeze(2)).sum().backward()
    assert (y.detach().squeeze(2) - T_(f["y"])).abs().max().item() < 1e-5
    assert (x.grad.squeeze(2) - T_(f["dx"])).abs().max().item() < 1e-4
    for n, p in m.named_parameters():
        ref = T_(f["d_" + n])
        assert (p.grad.reshape(ref.shape) - ref).abs().max().item() < 1e-4 * max(1.0, ref.abs().max().item()), n


@pytest.mark.parametrize("shape", [(1, 3, 5, 4, 6), (2, 4, 3, 7, 2)])
def test_h1_is_the_2d_op_with_time_as_the_column_axis(shape):
    B, Cq, C, T, W = shape
    q, k, v = _qkv(B, Cq, C, T, 1, W, seed=3)
    dout = torch.randn(B, C, T, 1, W, dtype=torch.float64)
    out, lse = O3.cca3d_forward(q, k, v)
    o2, l2 = O.cca_forward(q[:, :, :, 0], k[:, :, :, 0], v[:, :, :, 0])
    assert (out[:, :, :, 0] - o2).abs().max().item() < 1e-12 and (lse[:, :, 0] - l2).abs().max().item() < 1e-12
    g3 = O3.cca3d_backward(dout, q, k, v)
    g2 = O.cca_backward(dout[:, :, :, 0], q[:, :, :, 0], k[:, :, :, 0], v[:, :, :, 0])
    for a, b in zip(g3, g2):
        assert (a[:, :, :, 0] - b).abs().max().item() < 1e-12


def test_t1_backward_is_the_2d_backward_on_every_frame():
    q, k, v = _qkv(2, 3, 5, 1, 4, 6, seed=5)
    dout = torch.randn(2, 5, 1, 4, 6, dtype=torch.float64)
    for a, b in zip(O3.cca3d_backward(dout, q, k, v), O.cca_backward(dout[:, :, 0], q[:, :, 0], k[:, :, 0], v[:, :, 0])):
        assert (a[:, :, 0] - b).abs().max().item() < 1e-12


def test_3d_symbols_are_exported():
    lib = capi.load()
    for name in ("cca_b200_tc3d_supported", "cca_b200_workspace_bytes3d", "cca_b200_forward3d", "cca_b200_backward3d"):
        assert name in capi.SYMBOLS and getattr(lib, name) is not None
    assert lib.cca_b200_version() == 200                  # the 3D entry points are an addition to version 0.2.0


def test_3d_entry_points_reject_bad_arguments_before_any_cuda_call():
    lib = capi.load()
    nhwc = capi.CCA_FLAG_NHWC
    rc = lib.cca_b200_forward3d(None, None, None, None, None, None, 0, 1, 16, 64, 4, 5, 5, capi.CCA_F32, nhwc, None)
    assert rc == -1 and b"null" in lib.cca_b200_last_error()
    p = 16                                  # any non-null address: every check below comes before anything touches it
    for T in (0, -3):
        rc = lib.cca_b200_forward3d(p, p, p, p, p, p, 1 << 30, 1, 16, 64, T, 5, 5, capi.CCA_F32, nhwc, None)
        assert rc == -1 and b"dimension" in lib.cca_b200_last_error()
    rc = lib.cca_b200_forward3d(p, p, p, p, p, p, 1 << 30, 1, 16, 64, 4, 5, 5, 7, nhwc, None)
    assert rc == -1 and b"dtype" in lib.cca_b200_last_error()
    rc = lib.cca_b200_forward3d(p, p, p, p, p, p, 16, 1, 16, 64, 4, 5, 5, capi.CCA_F32, nhwc, None)
    assert rc == -3
    rc = lib.cca_b200_backward3d(p, p, p, p, p, p, p, p, p, p, 16, 1, 16, 64, 4, 5, 5, capi.CCA_F32, nhwc, None)
    assert rc == -3
    rc = lib.cca_b200_backward3d(p, p, p, None, p, p, p, p, p, p, 1 << 30, 1, 16, 64, 4, 5, 5, capi.CCA_F32, nhwc, None)
    assert rc == -1 and b"null" in lib.cca_b200_last_error()
    err = lib.cca_b200_last_error
    both = capi.CCA_FLAG_FORCE_SIMT | capi.CCA_FLAG_FORCE_TC
    for fn, n in ((lib.cca_b200_forward3d, 6), (lib.cca_b200_backward3d, 10)):
        def call(ptrs=(p,) * n, nbytes=1 << 30, B=1, T=4, dtype=capi.CCA_F32, flags=nhwc):
            return fn(*ptrs, nbytes, B, 16, 64, T, 5, 5, dtype, flags, None)
        assert call(ptrs=(p,) * (n - 1) + (None,)) == -1 and b"null" in err()
        assert call(B=0) == -1 and b"dimension" in err()
        assert call(T=0) == -1 and b"dimension" in err()
        assert call(dtype=7) == -1 and b"dtype" in err()
        assert call(flags=both) == -1 and b"exclusive" in err()
        assert call(flags=both | nhwc) == -1 and b"exclusive" in err()
        assert call(nbytes=16) == -3 and b"workspace" in err()


def _a16(x):
    return (x + 15) // 16 * 16


@pytest.mark.parametrize("shape", [(1, 64, 512, 8, 97, 97), (2, 16, 64, 3, 130, 20), (1, 32, 128, 32, 65, 65)])
def test_3d_workspace_sizes(shape):
    B, Cq, C, T, H, W = shape
    lib = capi.load()
    npix = B * T * H * W
    nparts = -(-H // 112) + -(-W // 112)
    fwd = lib.cca_b200_workspace_bytes3d(capi.CCA_WS_FORWARD, *shape, capi.CCA_F32, capi.CCA_FLAG_NHWC)
    assert fwd == _a16((nparts + 1) * npix * 4) + _a16(B * T * 4)        # lse planes (+ the time plane), per-frame counters
    bwd = lib.cca_b200_workspace_bytes3d(capi.CCA_WS_BACKWARD, *shape, capi.CCA_F32, capi.CCA_FLAG_NHWC)
    assert bwd == lib.cca_b200_workspace_bytes_ex(capi.CCA_WS_BACKWARD, B * T, Cq, C, H, W, capi.CCA_F32, capi.CCA_FLAG_NHWC)
    det = capi.CCA_FLAG_NHWC | capi.CCA_FLAG_DETERMINISTIC
    for which, base in ((capi.CCA_WS_FORWARD, fwd), (capi.CCA_WS_BACKWARD, bwd)):
        extra = lib.cca_b200_workspace_bytes3d(which, *shape, capi.CCA_F32, det) - base
        extra2d = (lib.cca_b200_workspace_bytes_ex(which, B * T, Cq, C, H, W, capi.CCA_F32, det)
                   - lib.cca_b200_workspace_bytes_ex(which, B * T, Cq, C, H, W, capi.CCA_F32, capi.CCA_FLAG_NHWC))
        assert extra == (extra2d if nparts > 2 else 0)                 # the 2D passes' planes; the time pass needs none
        assert lib.cca_b200_workspace_bytes3d(which, *shape, capi.CCA_BF16, det) == base
    assert lib.cca_b200_workspace_bytes3d(capi.CCA_WS_FORWARD, B, Cq, C, 0, H, W, capi.CCA_F32, 0) == 0


def test_3d_coverage_without_gpu():
    lib = capi.load()
    for T in (0, 33, 64):
        assert lib.cca_b200_tc3d_supported(capi.CCA_WS_FORWARD, 1, 64, 512, T, 9, 9, capi.CCA_F32) == 0
    assert lib.cca_b200_tc3d_supported(capi.CCA_WS_BACKWARD, 1, 8, 512, 4, 9, 9, capi.CCA_F32) == 0    # Cq = 8
    assert lib.cca_b200_tc3d_supported(capi.CCA_WS_FORWARD, 1, 64, 96, 4, 9, 9, capi.CCA_F32) == 0     # C % 64
    assert lib.cca_b200_tc3d_supported(capi.CCA_WS_FORWARD, 1, 64, 512, 4, 897, 9, capi.CCA_F32) == 0  # line > 896


def test_module_parameters_mirror_the_2d_module():
    from ccnet_b200 import CrissCrossAttention, CrissCrossAttention3D
    import cc_attention
    assert cc_attention.CrissCrossAttention3D is CrissCrossAttention3D
    m3, m2 = CrissCrossAttention3D(64), CrissCrossAttention(64)
    p3, p2 = dict(m3.named_parameters()), dict(m2.named_parameters())
    assert set(p3) == set(p2) == {"gamma", "query_conv.weight", "query_conv.bias", "key_conv.weight", "key_conv.bias",
                                  "value_conv.weight", "value_conv.bias"}
    assert p3["query_conv.weight"].shape == p3["key_conv.weight"].shape == (8, 64, 1, 1, 1)
    assert p3["value_conv.weight"].shape == (64, 64, 1, 1, 1)
    assert all(p3[n].shape[:2] == p2[n].shape[:2] for n in p3)
    assert torch.equal(m3.gamma, torch.zeros(1))
    with pytest.raises(RuntimeError, match="CUDA"):
        m3(torch.randn(1, 64, 2, 3, 3))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("Cq,C", [(64, 512), (8, 24)])
def test_fake_implementations_give_shapes_and_memory_formats(dtype, Cq, C):
    """channels_last_3d results where the tensor-core path runs (on an H100), contiguous ones where the generic kernels do"""
    import ccnet_b200  # noqa: F401  (registers torch.ops.cca)
    from ccnet_b200.functional import tc3d_eligible
    from torch._subclasses.fake_tensor import FakeTensorMode
    cl = tc3d_eligible(2, Cq, C, 5, 20, 30, dtype)
    if Cq == 8:
        assert not cl
    fmt = torch.channels_last_3d if cl else torch.contiguous_format
    with FakeTensorMode():
        q = torch.empty(2, Cq, 5, 20, 30, device="cuda", dtype=dtype)
        v = torch.empty(2, C, 5, 20, 30, device="cuda", dtype=dtype)
        out, lse = torch.ops.cca.forward3d(q, q, v)
        assert out.shape == v.shape and out.dtype == dtype and out.is_contiguous(memory_format=fmt)
        assert lse.shape == (2, 5, 20, 30) and lse.dtype == torch.float32
        grads = torch.ops.cca.backward3d(out, q, q, v, out, lse)
        assert [g.shape for g in grads] == [q.shape, q.shape, v.shape]
        assert all(g.dtype == dtype and g.is_contiguous(memory_format=fmt) for g in grads)


def test_generic_kernels_have_no_spills_and_no_stack(tmp_path):
    report = _ptxas(os.path.join(build.CSRC, "cca_simt_3d.cu"), tmp_path)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", report)
    # {forward, delta, backward} x {fp32, bf16, f16}
    assert len(frames) == 9 and all(f == ("0", "0", "0") for f in frames), frames


def _ptxas(src, tmp_path):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    out = subprocess.run([nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "k.o")],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    return out.stdout + out.stderr


def test_time_kernels_have_no_spills_and_no_stack(tmp_path):
    report = _ptxas(os.path.join(build.CSRC, "cca_tc_time.cu"), tmp_path)
    assert "C7514" not in report                          # (no wgmma here; nothing of the 2D kernels is compiled in this file)
    names, frames = [], []
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            names.append(m.group(1))
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            frames.append((names[-1], int(m.group(1)), int(m.group(2)), int(m.group(3))))
    # {stats, values, backward} x {T <= 8, 16, 32} x {fp32, bf16, f16}
    assert len(names) == 27 and all("cca_time_" in n for n in names), names
    assert len(frames) == 27 and all(f[1:] == (0, 0, 0) for f in frames), frames


def _branch_parts(q, k, v, dout):
    """{tensor: (column part, row part, time part)} of out, dq, dk, dv in fp64"""
    B, Cq, T, H, W = q.shape
    a = torch.softmax(O3.cca3d_logits(q, k), dim=4)
    ah, aw, at = a[..., :H], a[..., H:H + W], a[..., H + W:]
    o = (torch.einsum("bthwg,bctgw->bcthw", ah, v), torch.einsum("bthwg,bcthg->bcthw", aw, v),
         torch.einsum("bthws,bcshw->bcthw", at, v))
    delta = (dout * sum(o)).sum(1).unsqueeze(-1)
    dh = ah * (torch.einsum("bcthw,bctgw->bthwg", dout, v) - delta)
    dw = aw * (torch.einsum("bcthw,bcthg->bthwg", dout, v) - delta)
    dt = at * (torch.einsum("bcthw,bcshw->bthws", dout, v) - delta)
    dq = (torch.einsum("bthwg,bctgw->bcthw", dh, k), torch.einsum("bthwg,bcthg->bcthw", dw, k),
          torch.einsum("bthws,bcshw->bcthw", dt, k))
    dk = (torch.einsum("bthwg,bcthw->bctgw", dh, q), torch.einsum("bthwg,bcthw->bcthg", dw, q),
          torch.einsum("bthws,bcthw->bcshw", dt, q))
    dv = (torch.einsum("bthwg,bcthw->bctgw", ah, dout), torch.einsum("bthwg,bcthw->bcthg", aw, dout),
          torch.einsum("bthws,bcthw->bcshw", at, dout))
    return dict(out=o, dq=dq, dk=dk, dv=dv)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
def test_16bit_rounding_chain_of_the_native_3d_path(dtype):
    """The native 16-bit path rounds each output element three times: the column part is stored in the I/O type, the row
    part reduce-added onto it (rounded), the time part added by the time pass (rounded again).  The floor of that chain alone
    (exact P, dS; 16-bit inputs; max|err| / max(1, max|ref|)) decides the policy of functional._upcast: fp16 stays within
    a third of its budget (tests/f16_budget.py), bf16 reaches 0.73 of its 1e-2 budget, so bf16 with T > 1 runs on the fp32
    kernels and is rounded once (floor 2.9e-3 here, under half the budget)."""
    from f16_budget import F16_BUDGET
    rnd = lambda x: x.to(dtype).double()
    worst3, worst1 = {}, {}
    for shape in [(1, 64, 128, 4, 12, 10), (1, 32, 64, 8, 9, 11), (2, 16, 64, 3, 20, 15)]:
        B, Cq, C, T, H, W = shape
        g = torch.Generator().manual_seed(sum(shape))
        q, k = (rnd(torch.randn(B, Cq, T, H, W, generator=g, dtype=torch.float64) * 0.7) for _ in range(2))
        v, dout = (rnd(torch.randn(B, C, T, H, W, generator=g, dtype=torch.float64)) for _ in range(2))
        for n, (c, r, t) in _branch_parts(q, k, v, dout).items():
            ref = c + r + t
            s = max(1.0, ref.abs().max().item())
            worst3[n] = max(worst3.get(n, 0.0), (rnd(rnd(rnd(c) + r) + t) - ref).abs().max().item() / s)
            worst1[n] = max(worst1.get(n, 0.0), (rnd(ref) - ref).abs().max().item() / s)
    print(dtype, "three roundings", worst3, "one", worst1)
    if dtype == torch.float16:
        assert all(F16_BUDGET[n] >= 2.5 * e for n, e in worst3.items()), worst3
    else:
        assert max(worst3.values()) > 0.5e-2                   # within 2x of the budget: not run natively (T > 1)
        assert max(worst1.values()) <= 0.5e-2, worst1                # one rounding: the budget is >= 2x its floor


def test_bf16_with_time_runs_on_the_fp32_kernels():
    from ccnet_b200.functional import _upcast
    assert _upcast(torch.bfloat16, 9, 9, False, T=2) and not _upcast(torch.bfloat16, 9, 9, False, T=1)
    assert not _upcast(torch.float16, 97, 97, False, T=8) and _upcast(torch.float16, 97, 113, False, T=8)
    assert not _upcast(torch.float32, 200, 200, False, T=8)
