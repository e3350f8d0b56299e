"""CPU tests of the attention map (cc_attention/functions.py:40, `concate`): the oracle against the reference's own maps and
gradients (tests/golden/attn_*.npz) and fp64 autograd, the emulated kernel inside its budget, argument validation of the C
entry points before any CUDA call, and the new kernels' resources."""
import glob
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import attn_budget as AB
from ccnet_b200 import build, capi
from oracle.cca_oracle import CrissCrossAttentionOracle

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "attn_*.npz")))


def oracle_module_maps(f, dtype=torch.float64):
    """(module, x, [maps]) of the oracle module with the fixture's parameters; maps from the module's own convs"""
    C = f["x"].shape[1]
    m = CrissCrossAttentionOracle(C).to(dtype)
    m.load_state_dict({n[2:]: torch.from_numpy(f[n]).to(dtype) for n in f.files if n.startswith("p_")})
    x = torch.from_numpy(f["x"]).to(dtype).requires_grad_(True)
    y, maps = x, []
    for _ in range(int(f["R"])):
        maps.append(AB.attention_map(m.query_conv(y), m.key_conv(y)))
        y = m(y)
    return m, x, maps


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p) for p in FIXTURES])
def test_oracle_map_and_gradients_match_the_reference(path):
    f = np.load(path)
    m, x, maps = oracle_module_maps(f)
    loss = 0
    for i, a in enumerate(maps):
        ref = torch.from_numpy(f[f"A_{i}"]).double()
        assert a.shape == ref.shape
        assert (a - ref).abs().max().item() < 1e-6
        loss = loss + (a * torch.from_numpy(f[f"R_{i}"]).double()).sum()
    loss.backward()
    tol = lambda r: 1e-5 * max(1.0, np.abs(r).max())
    assert (x.grad.numpy() - f["dx"]).__abs__().max() < tol(f["dx"])
    for n, p in m.named_parameters():
        g = p.grad.numpy() if p.grad is not None else np.zeros(p.shape)
        assert np.abs(g - f["d_" + n]).max() < tol(f["d_" + n]), n
    if int(f["R"]) == 1:                    # one step: the map does not depend on v
        assert m.value_conv.weight.grad is None or not m.value_conv.weight.grad.any()


@pytest.mark.parametrize("shape", [(2, 8, 5, 6), (1, 4, 1, 11), (1, 4, 13, 1), (2, 16, 9, 7)])
def test_closed_form_backward_matches_fp64_autograd(shape):
    g = torch.Generator().manual_seed(1)
    q, k = (torch.randn(shape, generator=g, dtype=torch.float64).requires_grad_(True) for _ in range(2))
    a = AB.attention_map(q, k)
    assert a[..., :shape[2]].diagonal(dim1=1, dim2=3).abs().max() == 0          # self entries exactly 0
    assert torch.allclose(a.sum(-1), torch.ones_like(a.sum(-1)))
    r = torch.randn(a.shape, generator=g, dtype=torch.float64)
    gq, gk = torch.autograd.grad((a * r).sum(), (q, k))
    dq, dk = AB.attention_map_backward(r, q.detach(), k.detach())
    assert torch.allclose(dq, gq, atol=1e-12) and torch.allclose(dk, gk, atol=1e-12)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_emulated_kernel_is_inside_its_budget_and_a_dropped_term_is_not(dtype):
    g = torch.Generator().manual_seed(2)
    q, k = ((torch.randn(1, 32, 9, 11, generator=g) * 0.7).to(dtype) for _ in range(2))
    da = torch.randn(1, 9, 11, 20, generator=g)
    ref = AB.reference(q, k, da)
    emu = AB.emulate(q, k, da, dtype)
    bud = AB.budget(emu, ref, dtype)
    AB.check(emu, ref, bud)
    bad = dict(emu, dq=emu["dq"] * (1 + 8 * max(bud["dq"], 1e-3)))
    with pytest.raises(AssertionError):
        AB.check(bad, ref, bud)


def test_attention_entry_points_reject_bad_arguments_before_any_cuda_call():
    lib = capi.load()
    rc = lib.cca_b200_attention_forward(None, None, None, None, 0, 1, 16, 4, 4, capi.CCA_F32, 0, None)
    assert rc == -1 and b"null" in lib.cca_b200_last_error()
    rc = lib.cca_b200_attention_forward(None, None, None, None, 0, 0, 16, 4, 4, capi.CCA_F32, 0, None)
    assert rc == -1
    rc = lib.cca_b200_attention_forward(None, None, None, None, 0, 1, 16, 4, 4, 7, 0, None)
    assert rc == -1 and b"dtype" in lib.cca_b200_last_error()
    rc = lib.cca_b200_attention_backward(None, None, None, None, None, None, None, 0, 1, 16, 4, 4, capi.CCA_F32, 0, None)
    assert rc == -1 and b"null" in lib.cca_b200_last_error()
    p = 16                                  # any non-null address: the workspace check comes before anything touches it
    rc = lib.cca_b200_attention_backward(p, p, p, p, p, p, p, 0, 1, 16, 4, 4, capi.CCA_F32, 0, None)
    assert rc == -3
    rc = lib.cca_b200_attention_forward(p, p, p, p, 1 << 20, 2, 16, 1 << 16, 1 << 16, capi.CCA_F32, 0, None)
    assert rc == -2                         # map past 2^40 elements
    rc = lib.cca_b200_attention_forward(p, p, p + 2, p, 1 << 20, 1, 16, 4, 4, capi.CCA_F32, 0, None)
    assert rc == -1 and b"aligned" in lib.cca_b200_last_error()       # attn not even float-aligned
    rc = lib.cca_b200_attention_backward(p + 2, p, p, p, p, p, p, 1 << 20, 1, 16, 4, 4, capi.CCA_F32, 0, None)
    assert rc == -1 and b"aligned" in lib.cca_b200_last_error()
    err, big = lib.cca_b200_last_error, 1 << 30
    both = capi.CCA_FLAG_FORCE_SIMT | capi.CCA_FLAG_FORCE_TC
    for fn, n in ((lib.cca_b200_attention_forward, 4), (lib.cca_b200_attention_backward, 7)):
        def call(ptrs=(p,) * n, nbytes=big, B=1, Cq=16, dtype=capi.CCA_F32, flags=0):
            return fn(*ptrs, nbytes, B, Cq, 4, 4, dtype, flags, None)
        assert call(ptrs=(p,) * (n - 1) + (None,)) == -1 and b"null" in err()
        assert call(B=0) == -1 and b"dimension" in err()
        assert call(Cq=-16) == -1 and b"dimension" in err()
        assert call(dtype=7) == -1 and b"dtype" in err()
        assert call(flags=both) == -1 and b"exclusive" in err()
        assert call(flags=both | capi.CCA_FLAG_NHWC) == -1 and b"exclusive" in err()
        assert call(nbytes=0) == -3 and b"workspace" in err()


def test_attention_workspace_and_coverage_without_gpu():
    lib = capi.load()
    px = 8 * 97 * 97
    assert lib.cca_b200_attention_workspace_bytes(0, 8, 64, 97, 97, capi.CCA_F32, 0) == px * 8 + 32    # statistics planes
    assert lib.cca_b200_attention_workspace_bytes(1, 8, 64, 97, 97, capi.CCA_F32, 0) == (px * 4 + 255) // 256 * 256
    det = capi.CCA_FLAG_DETERMINISTIC | capi.CCA_FLAG_NHWC
    extra = (lib.cca_b200_attention_workspace_bytes(1, 1, 16, 193, 193, capi.CCA_F32, det)
             - lib.cca_b200_attention_workspace_bytes(1, 1, 16, 193, 193, capi.CCA_F32, capi.CCA_FLAG_NHWC))
    assert extra >= 2 * 4 * 193 * 193 * 16 * 4                     # dQ and dK planes, 4 partial planes each
    assert lib.cca_b200_attention_tc_supported(1, 8, 97, 97, capi.CCA_F32) == 0
    assert lib.cca_b200_attention_tc_supported(1, 64, 896, 897, capi.CCA_BF16) == 0


def _ptxas(src, tmp_path):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    out = subprocess.run([nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "k.o")],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    return out.stdout + out.stderr


def test_map_kernels_have_no_spills_and_no_serialised_wgmma(tmp_path):
    report = _ptxas(os.path.join(build.CSRC, "cca_tc_attn.cu"), tmp_path)
    assert "C7514" not in report, [l for l in report.splitlines() if "C7514" in l][:3]
    names, spills = [], []
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            names.append(m.group(1))
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            spills.append((names[-1], int(m.group(1)), int(m.group(2))))
    attn = [n for n in names if "cca_tc_attn" in n]
    # forward <80, 112> x <fp32, bf16, f16>; backward the same + the fp32 planes mode
    assert len([n for n in attn if "attn_fwd" in n]) == 6 and len([n for n in attn if "attn_bwd" in n]) == 8, attn
    assert all(s == 0 and l == 0 for _, s, l in spills), spills


def test_generic_map_kernels_have_no_spills(tmp_path):
    report = _ptxas(os.path.join(build.CSRC, "cca_simt_attn.cu"), tmp_path)
    names, spills = [], []
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            names.append(m.group(1))
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            spills.append((names[-1], int(m.group(1)), int(m.group(2))))
    # map, dq, dk for fp32 / bf16 / f16, and the rho pass
    assert len(names) == 10, names
    assert len(spills) == 10 and all(s == 0 and l == 0 for _, s, l in spills), spills
