"""CPU tests of causal criss-cross attention over clips (CCA_FLAG_CAUSAL) and its streaming step: the fp64 oracle
(tests/cca3d_causal_oracle.py) and its ties to tests/cca3d_oracle.py; the C entry points' flag, symbols, workspace sizes and
validation; the step's coverage; the fake implementations; the module's parameters; and the ptxas resources of the causal and
step kernels."""
import os
import re
import subprocess

import pytest
import torch

import cca3d_causal_oracle as OC
import cca3d_oracle as O3
from ccnet_b200 import build, capi
from oracle import cca_oracle as O


def _qkv(B, Cq, C, T, H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    mk = lambda c: torch.randn(B, c, T, H, W, generator=g, dtype=torch.float64)
    return mk(Cq), mk(Cq), mk(C)


SHAPES = [(1, 2, 3, 4, 3, 5), (2, 3, 2, 3, 4, 2), (1, 2, 3, 5, 1, 4), (1, 1, 2, 2, 2, 1)]


@pytest.mark.parametrize("shape", SHAPES)
def test_causal_logits_are_the_bidirectional_logits_with_future_time_keys_masked(shape):
    q, k, _ = _qkv(*shape)
    B, Cq, C, T, H, W = shape
    e, ec = O3.cca3d_logits(q, k), OC.cca3d_causal_logits(q, k)
    future = torch.ones(T, T, dtype=torch.bool).triu(1).view(1, T, 1, 1, T)
    et = e[..., H + W:].masked_fill(future, float("-inf"))
    assert torch.equal(ec[..., :H + W], e[..., :H + W]) and torch.equal(ec[..., H + W:], et)


@pytest.mark.parametrize("shape", [(1, 2, 3, 1, 3, 4), (2, 3, 2, 1, 5, 2)])
def test_at_t1_causal_is_the_bidirectional_op(shape):
    q, k, v = _qkv(*shape, seed=1)
    dout = torch.randn_like(v)
    for a, b in zip(OC.cca3d_causal_forward(q, k, v), O3.cca3d_forward(q, k, v)):
        assert (a - b).abs().max().item() < 1e-12
    for a, b in zip(OC.cca3d_causal_backward(dout, q, k, v), O3.cca3d_backward(dout, q, k, v)):
        assert (a - b).abs().max().item() < 1e-12


@pytest.mark.parametrize("shape", SHAPES)
def test_frame_0_is_the_2d_op_map_rows_sum_to_1_masked_entries_are_0(shape):
    q, k, v = _qkv(*shape, seed=2)
    B, Cq, C, T, H, W = shape
    out, lse = OC.cca3d_causal_forward(q, k, v)
    o2, l2 = O.cca_forward(q[:, :, 0], k[:, :, 0], v[:, :, 0])
    assert (out[:, :, 0] - o2).abs().max().item() < 1e-12 and (lse[:, 0] - l2).abs().max().item() < 1e-12
    a = OC.cca3d_causal_attention(q, k)
    assert (a.sum(-1) - 1).abs().max().item() < 1e-12
    assert (a[..., H + W:][OC.time_mask(T).view(1, T, 1, 1, T).expand(B, T, H, W, T)] == 0).all()
    assert (a[..., :H][torch.eye(H, dtype=torch.bool).view(1, 1, H, 1, H).expand(B, T, H, W, H)] == 0).all()


@pytest.mark.parametrize("shape", SHAPES)
def test_closed_form_gradients_match_autograd(shape):
    q, k, v = _qkv(*shape, seed=3)
    dout, dattn = torch.randn_like(v), torch.randn(*OC.cca3d_causal_logits(q, k).shape, dtype=torch.float64)
    qa, ka, va = (t.clone().requires_grad_(True) for t in (q, k, v))
    out, _ = OC.cca3d_causal_forward(qa, ka, va)
    ref = torch.autograd.grad(out, (qa, ka, va), dout)
    for a, b in zip(OC.cca3d_causal_backward(dout, q, k, v), ref):
        assert (a - b).abs().max().item() < 1e-10
    attn = OC.cca3d_causal_attention(qa, ka)
    ref = torch.autograd.grad(attn, (qa, ka), dattn)
    for a, b in zip(OC.cca3d_causal_attention_backward(dattn, q, k), ref):
        assert (a - b).abs().max().item() < 1e-10


@pytest.mark.parametrize("S", [0, 1, 4])
def test_step_oracle_is_the_last_frame_of_the_clip_oracle(S):
    q, k, v = _qkv(2, 3, 4, S + 1, 3, 5, seed=4 + S)
    out, lse = OC.cca3d_causal_forward(q, k, v)
    so, sl = OC.cca3d_step(q[:, :, S], k[:, :, S], v[:, :, S], k[:, :, :S], v[:, :, :S])
    assert (so - out[:, :, S]).abs().max().item() < 1e-12 and (sl - lse[:, S]).abs().max().item() < 1e-12


def test_flag_value_and_new_symbols():
    lib = capi.load()
    assert capi.CCA_FLAG_CAUSAL == 16
    hdr = open(os.path.join(build.HERE, "..", "include", "cca_b200.h")).read()
    assert re.search(r"#define CCA_FLAG_CAUSAL 16u", hdr)
    for name in ("cca_b200_forward3d_step", "cca_b200_workspace_bytes3d_step"):
        assert name in capi.SYMBOLS and name in hdr and getattr(lib, name) is not None
    assert lib.cca_b200_version() == 200                  # an addition to version 0.2.0


@pytest.mark.parametrize("shape", [(1, 64, 512, 8, 97, 97), (2, 16, 64, 3, 130, 20), (1, 32, 128, 32, 65, 65), (2, 8, 24, 40, 5, 7)])
def test_workspace_sizes_with_the_flag_equal_those_without_it(shape):
    lib = capi.load()
    C = capi.CCA_FLAG_CAUSAL
    for dt in (capi.CCA_F32, capi.CCA_BF16, capi.CCA_F16):
        for flags in (0, capi.CCA_FLAG_NHWC, capi.CCA_FLAG_NHWC | capi.CCA_FLAG_DETERMINISTIC, capi.CCA_FLAG_DETERMINISTIC):
            for which in (capi.CCA_WS_FORWARD, capi.CCA_WS_BACKWARD):
                assert (lib.cca_b200_workspace_bytes3d(which, *shape, dt, flags | C)
                        == lib.cca_b200_workspace_bytes3d(which, *shape, dt, flags))
            B, Cq, _, T, H, W = shape
            for bwd in (0, 1):
                assert (lib.cca_b200_attention_workspace_bytes3d(bwd, B, Cq, T, H, W, dt, flags | C)
                        == lib.cca_b200_attention_workspace_bytes3d(bwd, B, Cq, T, H, W, dt, flags))


@pytest.mark.parametrize("shape", [(1, 64, 512, 97, 97), (2, 16, 64, 130, 20), (3, 8, 24, 5, 7)])
def test_step_workspace_is_the_one_frame_forward_workspace(shape):
    B, Cq, C, H, W = shape
    lib = capi.load()
    for dt in (capi.CCA_F32, capi.CCA_BF16):
        for flags in (0, capi.CCA_FLAG_NHWC, capi.CCA_FLAG_NHWC | capi.CCA_FLAG_DETERMINISTIC):
            one = lib.cca_b200_workspace_bytes3d(capi.CCA_WS_FORWARD, B, Cq, C, 1, H, W, dt, flags)
            assert one > 0
            for S in (0, 7, 31, 40):
                assert lib.cca_b200_workspace_bytes3d_step(B, Cq, C, S, H, W, dt, flags) == one
    assert lib.cca_b200_workspace_bytes3d_step(B, Cq, C, -1, H, W, capi.CCA_F32, 0) == 0
    assert lib.cca_b200_workspace_bytes3d_step(0, Cq, C, 3, H, W, capi.CCA_F32, 0) == 0


def test_step_rejects_bad_arguments_before_any_cuda_call():
    lib = capi.load()
    err = lib.cca_b200_last_error
    p, nhwc = 16, capi.CCA_FLAG_NHWC
    both = capi.CCA_FLAG_FORCE_SIMT | capi.CCA_FLAG_FORCE_TC

    def call(ptrs=(p,) * 8, nbytes=1 << 30, B=1, S=3, dtype=capi.CCA_F32, flags=nhwc, Cq=16):
        return lib.cca_b200_forward3d_step(*ptrs, nbytes, B, Cq, 64, S, 5, 5, dtype, flags, None)
    assert call(S=-1) == -1 and b"negative" in err()
    assert call(B=0) == -1 and b"dimension" in err()
    assert call(Cq=0) == -1 and b"dimension" in err()
    assert call(dtype=7) == -1 and b"dtype" in err()
    for i in range(8):
        ptrs = [p] * 8
        ptrs[i] = None
        assert call(ptrs=tuple(ptrs)) == -1 and b"null" in err(), i
    assert call(nbytes=16) == -3 and b"workspace" in err()
    assert call(flags=both) == -1 and b"exclusive" in err()
    # S = 0: the caches are not read and may be NULL -- the call passes the pointer checks and stops at the workspace check
    # (which comes after them, before anything touches a device)
    rc = lib.cca_b200_forward3d_step(p, p, p, None, None, p, p, p, 16, 1, 16, 64, 0, 5, 5, capi.CCA_F32, nhwc, None)
    assert rc == -3 and b"workspace" in err()
    rc = lib.cca_b200_forward3d_step(p, p, p, None, p, p, p, p, 16, 1, 16, 64, 1, 5, 5, capi.CCA_F32, nhwc, None)
    assert rc == -1 and b"null" in err()


def test_step_plans_the_tensor_cores_by_the_coverage_of_a_clip_of_s_plus_1_frames(monkeypatch):
    """cca3d_step asks cca_b200_tc3d_supported about a clip of S + 1 frames (S <= 31 on tensor cores); recorded here
    without a device by stopping the call at its plan"""
    import ccnet_b200.functional as F_
    from torch._subclasses.fake_tensor import FakeTensorMode
    asked = []

    def plan(impl, det, covered, q, v=None, causal=False):
        asked.append(covered)
        raise RuntimeError("stop at the plan")
    monkeypatch.setattr(F_, "_plan", plan)
    lib = capi.load()
    with FakeTensorMode():
        for S in (0, 7, 31, 32):
            q, v = torch.empty(1, 16, 9, 9, device="cuda"), torch.empty(1, 64, 9, 9, device="cuda")
            kc, vc = torch.empty(1, 16, S, 9, 9, device="cuda"), torch.empty(1, 64, S, 9, 9, device="cuda")
            with pytest.raises(RuntimeError, match="stop at the plan"):
                F_.cca3d_step(q, q, v, kc, vc)
    calls = []
    real = lib.cca_b200_tc3d_supported
    monkeypatch.setattr(lib, "cca_b200_tc3d_supported", lambda *a: calls.append(a) or real(*a), raising=False)
    for covered in asked:
        covered()
    assert [c[4] for c in calls] == [1, 8, 32, 33]                        # T = S + 1
    assert all(c[:4] == (capi.CCA_WS_FORWARD, 1, 16, 64) and c[5:] == (9, 9, capi.CCA_F32) for c in calls), calls


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("Cq,C", [(64, 512), (8, 24)])
def test_fake_implementations_give_shapes_and_memory_formats(dtype, Cq, C):
    import ccnet_b200  # noqa: F401
    from ccnet_b200.functional import tc3d_eligible
    from torch._subclasses.fake_tensor import FakeTensorMode
    cl = tc3d_eligible(2, Cq, C, 5, 20, 30, dtype)
    fmt = torch.channels_last_3d if cl else torch.contiguous_format
    with FakeTensorMode():
        q = torch.empty(2, Cq, 5, 20, 30, device="cuda", dtype=dtype)
        v = torch.empty(2, C, 5, 20, 30, device="cuda", dtype=dtype)
        out, lse = torch.ops.cca.forward3d(q, q, v, True)
        assert out.shape == v.shape and out.dtype == dtype and out.is_contiguous(memory_format=fmt)
        assert lse.shape == (2, 5, 20, 30) and lse.dtype == torch.float32
        grads = torch.ops.cca.backward3d(out, q, q, v, out, lse, True)
        assert [g.shape for g in grads] == [q.shape, q.shape, v.shape]
        assert all(g.dtype == dtype and g.is_contiguous(memory_format=fmt) for g in grads)
        attn = torch.ops.cca.attention3d(q, q, "auto", True)
        assert attn.shape == (2, 5, 20, 30, 20 + 30 + 5) and attn.dtype == torch.float32
        dq, dk = torch.ops.cca.attention3d_backward(attn, attn, q, q, "auto", True)
        assert dq.shape == dk.shape == q.shape
        # the step: the new frame [B,c,H,W] and caches of S = 4 frames
        q2, v2 = q[:, :, 0], v[:, :, 0]
        o, l = torch.ops.cca.forward3d_step(q2, q2, v2, q[:, :, :4], v[:, :, :4])
        fmt2 = torch.channels_last if tc3d_eligible(2, Cq, C, 5, 20, 30, dtype) else torch.contiguous_format
        assert o.shape == v2.shape and o.dtype == dtype and o.is_contiguous(memory_format=fmt2)
        assert l.shape == (2, 20, 30) and l.dtype == torch.float32


def test_causal_module_has_the_parameters_of_the_bidirectional_module():
    from ccnet_b200 import CrissCrossAttention3D
    m, mc = CrissCrossAttention3D(64), CrissCrossAttention3D(64, causal=True)
    assert mc.causal and not m.causal
    assert {n: p.shape for n, p in m.named_parameters()} == {n: p.shape for n, p in mc.named_parameters()}
    assert list(m.state_dict()) == list(mc.state_dict())
    mc.load_state_dict(m.state_dict())
    with pytest.raises(RuntimeError, match="causal"):
        m.step(torch.randn(1, 64, 3, 3))
    with pytest.raises(RuntimeError, match="CUDA"):
        mc.step(torch.randn(1, 64, 3, 3))


def test_step_refuses_inputs_that_require_grad():
    from ccnet_b200 import cca3d_step
    q = torch.randn(1, 2, 3, 3, requires_grad=True)
    with pytest.raises(RuntimeError, match="causal=True"):
        cca3d_step(q, q, q, q.unsqueeze(2), q.unsqueeze(2))


def _ptxas(src, tmp_path):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    out = subprocess.run([nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "k.o")],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    report = out.stdout + out.stderr
    names, frames = [], []
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            names.append(m.group(1))
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            frames.append((names[-1], int(m.group(1)), int(m.group(2)), int(m.group(3))))
    return report, names, frames


def test_causal_tensor_core_time_kernels_have_no_spills_and_no_stack(tmp_path):
    report, names, frames = _ptxas(os.path.join(build.CSRC, "cca_tc_causal.cu"), tmp_path)
    assert "C7514" not in report                          # no wgmma in this file
    # {stats, values, backward, map forward, map backward} x {T <= 8, 16, 32} x 3 dtypes + {step stats, step values} x 3
    assert len(names) == 51 and all("cca_time_" in n for n in names), names
    assert len(frames) == 51 and all(f[1:] == (0, 0, 0) for f in frames), frames


def test_causal_generic_kernels_have_no_stack_but_the_16bit_forward(tmp_path):
    """ptxas spills 24 bytes in the 16-bit causal forward (40 registers; the bidirectional kernel of the same body has 48 and
    none): a few loads per pixel on the generic path, pinned here so that a change shows"""
    _, names, frames = _ptxas(os.path.join(build.CSRC, "cca_simt_causal.cu"), tmp_path)
    # {forward, delta, backward, map, map dq, map dk, step} x 3 dtypes
    assert len(names) == 21 and len(frames) == 21, names
    spilled = {f[0] for f in frames if f[1:] != (0, 0, 0)}
    assert all("causal_fwd_kernel" in n and ("__nv_bfloat16" in n or "__half" in n) for n in spilled), spilled
    assert all(f[1:] == (16, 24, 24) for f in frames if f[0] in spilled), frames
