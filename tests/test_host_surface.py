"""CPU tests: the C-ABI library loads and exports every symbol of include/cca_b200.h, the
nn.Module mirrors the reference surface, and nothing silently falls back to CPU."""
import ctypes
import json
import os
import re

import pytest
import torch

import cc_attention
import ccnet_b200
from ccnet_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "cca_b200.h")).read()
    declared = set(re.findall(r"CCA_API[^;(]*?\b(cca_b200_\w+)\s*\(", hdr))
    assert declared == set(capi.SYMBOLS), declared ^ set(capi.SYMBOLS)
    lib = ctypes.CDLL(capi.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), name


def test_version_and_workspace_and_strerror_without_gpu():
    lib = capi.load()
    assert lib.cca_b200_version() == 200
    px = 8 * 97 * 97
    # forward: two partial-lse planes (row + column) + 8 zero-ahead counters; backward: delta + 3 x 8 counters
    assert lib.cca_b200_workspace_bytes(capi.CCA_WS_FORWARD, 8, 64, 512, 97, 97, capi.CCA_F32) == px * 8 + 32
    assert lib.cca_b200_workspace_bytes(capi.CCA_WS_BACKWARD, 8, 64, 512, 97, 97, capi.CCA_F32) == px * 4 + 96
    # lines longer than 112 pixels are tiled: one plane per key block
    assert lib.cca_b200_workspace_bytes(capi.CCA_WS_FORWARD, 1, 64, 512, 193, 193, capi.CCA_F32) == 193 * 193 * 16 + 16
    assert lib.cca_b200_tc_supported(capi.CCA_WS_FORWARD, 1, 8, 64, 32, 32, capi.CCA_F32) == 0      # Cq < 16
    assert lib.cca_b200_strerror(0) == b"ok"
    assert b"unsupported" in lib.cca_b200_strerror(-2)


def _workspace_cases():
    with open(os.path.join(ROOT, "tests", "golden", "workspace_bytes.json")) as f:
        return sorted(json.load(f).items())


@pytest.mark.parametrize("query,cases", _workspace_cases(), ids=lambda x: x if isinstance(x, str) else "")
def test_workspace_bytes_match_the_recorded_sizes(query, cases):
    # callers allocate by these sizes: every one stays byte-identical (fixture: tests/golden/make_workspace_bytes.py)
    fn = getattr(capi.load(), query)
    wrong = [(args, want, fn(*args)) for *args, want in cases if fn(*args) != want]
    assert not wrong, f"{len(wrong)} of {len(cases)} sizes differ, e.g. {wrong[:5]}"


def test_invalid_arguments_are_rejected_before_any_cuda_call():
    lib = capi.load()
    rc = lib.cca_b200_forward(None, None, None, None, None, None, 0, 1, 8, 64, 4, 4, 0, 0, None)
    assert rc == -1 and b"null" in lib.cca_b200_last_error()
    rc = lib.cca_b200_forward(None, None, None, None, None, None, 0, 0, 8, 64, 4, 4, 0, 0, None)
    assert rc == -1
    rc = lib.cca_b200_forward(None, None, None, None, None, None, 0, 1, 8, 64, 4, 4, 7, 0, None)
    assert rc == -1 and b"dtype" in lib.cca_b200_last_error()
    err = lib.cca_b200_last_error
    p, big = 16, 1 << 30                    # any non-null address: every check below comes before anything touches it
    both = capi.CCA_FLAG_FORCE_SIMT | capi.CCA_FLAG_FORCE_TC
    for fn, n in ((lib.cca_b200_forward, 6), (lib.cca_b200_backward, 10)):
        def call(ptrs=(p,) * n, nbytes=big, B=1, dtype=capi.CCA_F32, flags=0):
            return fn(*ptrs, nbytes, B, 8, 64, 4, 4, dtype, flags, None)
        assert call(ptrs=(None,) * n) == -1 and b"null" in err()
        assert call(ptrs=(p,) * (n - 1) + (None,)) == -1 and b"null" in err()
        assert call(B=0) == -1 and b"dimension" in err()
        assert call(B=-2) == -1 and b"dimension" in err()
        assert call(dtype=7) == -1 and b"dtype" in err()
        assert call(flags=both) == -1 and b"exclusive" in err()
        assert call(flags=both | capi.CCA_FLAG_NHWC) == -1 and b"exclusive" in err()
        assert call(nbytes=16) == -3 and b"workspace" in err()


def test_projection_gemms_reject_bad_arguments_before_any_cuda_call():
    lib = capi.load()
    err = lib.cca_b200_last_error
    p, big = 16, 1 << 30                    # any non-null address: every check below comes before anything touches it
    det = capi.CCA_FLAG_DETERMINISTIC
    # name -> (pointer count, call(pointers, workspace bytes, pixels, C, Cq))
    gemms = {
        "project": (11, lambda ptrs, nb, px, C, Cq: lib.cca_b200_qkv_project(*ptrs, nb, px, C, Cq, None)),
        "dgrad": (9, lambda ptrs, nb, px, C, Cq: lib.cca_b200_qkv_project_dgrad(*ptrs, nb, px, C, Cq, 0, None)),
        "wgrad": (9, lambda ptrs, nb, px, C, Cq: lib.cca_b200_qkv_project_wgrad(*ptrs, px, C, Cq, None)),
        "wgrad_ex": (9, lambda ptrs, nb, px, C, Cq: lib.cca_b200_qkv_project_wgrad_ex(*ptrs, px, C, Cq, p, nb, det, None)),
    }
    for name, (n, fn) in gemms.items():
        def call(ptrs=(p,) * n, nbytes=big, px=64, C=64, Cq=64):
            return fn(ptrs, nbytes, px, C, Cq)
        assert call(ptrs=(None,) + (p,) * (n - 1)) == -1 and b"null" in err(), name
        assert call(ptrs=(None,) * n, px=0) == -1 and b"null" in err(), name          # (null pointers are checked first)
        for px, C, Cq in ((0, 64, 64), (-1, 64, 64), (1 << 31, 64, 64), (64, 0, 64), (64, 64, 0), (64, -64, 64)):
            assert call(px=px, C=C, Cq=Cq) == -1 and b"dimension" in err(), (name, px, C, Cq)
    for name in ("project", "dgrad"):
        n, fn = gemms[name]
        assert fn((p,) * n, 16, 64, 64, 64) == -3 and b"workspace" in err(), name
        assert fn((p,) * (n - 1) + (None,), big, 64, 64, 64) == -1 and b"null" in err(), name    # the workspace
    assert gemms["dgrad"][1]((p,) * 6 + (None, p, p), big, 0, 64, 64) == -1 and b"dimension" in err()   # scale may be NULL
    assert gemms["wgrad"][1]((p,) * 8 + (None,), big, 0, 64, 64) == -1 and b"dimension" in err()       # db may be NULL
    # the deterministic weight gradient needs its workspace; without the flag it may be NULL
    assert lib.cca_b200_qkv_project_wgrad_ex(*(p,) * 9, 64, 64, 64, None, 0, det, None) == -1 and b"null" in err()
    assert lib.cca_b200_qkv_project_wgrad_ex(*(p,) * 9, 0, 64, 64, None, 0, 0, None) == -1 and b"dimension" in err()


def test_module_surface_matches_reference():
    m = cc_attention.CrissCrossAttention(512)
    assert isinstance(m, ccnet_b200.CrissCrossAttention)
    shapes = {n: tuple(p.shape) for n, p in m.named_parameters()}
    assert shapes == {
        "gamma": (1,),
        "query_conv.weight": (64, 512, 1, 1), "query_conv.bias": (64,),
        "key_conv.weight": (64, 512, 1, 1), "key_conv.bias": (64,),
        "value_conv.weight": (512, 512, 1, 1), "value_conv.bias": (512,),
    }
    assert float(m.gamma) == 0.0                       # functions.py:24
    assert sum(p.numel() for p in m.parameters()) == 328321  # 2*(64*512+64) + 512*512+512 + 1
    assert hasattr(m, "softmax") and hasattr(m, "INF")  # functions.py:22-23


def test_state_dict_roundtrip_with_oracle_module():
    from oracle.cca_oracle import CrissCrossAttentionOracle
    ref = CrissCrossAttentionOracle(64)
    m = cc_attention.CrissCrossAttention(64)
    missing, unexpected = m.load_state_dict(ref.state_dict(), strict=False)
    assert not missing and not unexpected


def test_no_cpu_fallback():
    m = cc_attention.CrissCrossAttention(64)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.randn(1, 64, 4, 4))
    with pytest.raises(RuntimeError, match="CUDA"):
        ccnet_b200.cca_forward(torch.randn(1, 8, 4, 4), torch.randn(1, 8, 4, 4), torch.randn(1, 64, 4, 4))


def test_product_does_not_import_oracle():
    for root, _, files in os.walk(os.path.join(ROOT, "ccnet_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(root, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, f
    assert "oracle" not in open(os.path.join(ROOT, "cc_attention", "__init__.py")).read().replace("oracle/", "")


def test_torch_ops_are_registered_with_fake_implementations():
    """SURVEY 8(b): torch.ops.cca.{forward, backward, forward_residual} exist and shape-infer under FakeTensorMode, so a
    traced / compiled networks/ccnet.py does not graph-break on the operator."""
    from torch._subclasses.fake_tensor import FakeTensorMode
    assert all(hasattr(torch.ops.cca, n) for n in ("forward", "backward", "forward_residual"))
    with FakeTensorMode():
        q = torch.empty(2, 8, 5, 6, device="cuda")
        v = torch.empty(2, 64, 5, 6, device="cuda")
        out, lse = torch.ops.cca.forward(q, q, v)
        assert out.shape == v.shape and out.dtype == v.dtype and lse.shape == (2, 5, 6) and lse.dtype == torch.float32
        dq, dk, dv = torch.ops.cca.backward(out, q, q, v, out, lse)
        assert dq.shape == q.shape and dv.shape == v.shape
        y, lse2, o2 = torch.ops.cca.forward_residual(q, q, v, v, torch.empty(1, device="cuda"))
        assert y.shape == v.shape and lse2.shape == lse.shape and o2.shape == v.shape
    torch.library.opcheck  # noqa: B018  (present in this torch; the GPU suite runs it on real tensors)


def test_differentiable_ops_end_in_their_mode_arguments():
    """the eight differentiable-op schemas end in the call's mode, impl and deterministic appended after the arguments they
    had, so positional calls keep their meaning; under FakeTensorMode those calls still work, and impl lands where the
    fakes read it: impl="tc" on a shape the tensor-core kernels do not cover raises, as the real call does"""
    from torch._subclasses.fake_tensor import FakeTensorMode
    mode2d = [("impl", "auto"), ("deterministic", None)]
    tails = {"forward": mode2d, "backward": mode2d, "attention": mode2d, "attention_backward": mode2d,
             "forward3d": [("causal", False), ("window", 0)] + mode2d,
             "backward3d": [("causal", False), ("window", 0)] + mode2d,
             "attention3d": [("impl", "auto"), ("causal", False), ("window", 0), ("deterministic", None)],
             "attention3d_backward": [("impl", "auto"), ("causal", False), ("window", 0), ("deterministic", None)]}
    for name, tail in tails.items():
        args = getattr(torch.ops.cca, name).default._schema.arguments
        assert [(a.name, a.default_value) for a in args[-len(tail):]] == tail, name
        assert str(args[-1].type) == "Optional[bool]" and not any(a.kwarg_only for a in args), name
    with FakeTensorMode():
        q = torch.empty(2, 16, 5, 20, 30, device="cuda")
        v = torch.empty(2, 64, 5, 20, 30, device="cuda")
        out, lse = torch.ops.cca.forward3d(q, q, v, True, 3)
        grads = torch.ops.cca.backward3d(out, q, q, v, out, lse, True, 3)
        attn = torch.ops.cca.attention3d(q, q, "auto", True, 3)
        dq, dk = torch.ops.cca.attention3d_backward(attn, attn, q, q, "auto", True, 3)
        o, l = torch.ops.cca.forward3d_step(q[:, :, 0], q[:, :, 0], v[:, :, 0], q, v, 4, 1)
        assert [t.shape for t in (out, lse, *grads, attn, dq, dk, o, l)] == [
            v.shape, (2, 5, 20, 30), q.shape, q.shape, v.shape, (2, 5, 20, 30, 55), q.shape, q.shape, v[:, :, 0].shape,
            (2, 20, 30)]
        with pytest.raises(ValueError):
            torch.ops.cca.forward3d(q, q, v, False, 3)
        # Cq = 8, C = 24: a shape the tensor-core kernels do not cover on any machine
        q, v = torch.empty(2, 8, 5, 20, 30, device="cuda"), torch.empty(2, 24, 5, 20, 30, device="cuda")
        out, lse = torch.ops.cca.forward3d(q, q, v, True, 3)
        attn = torch.ops.cca.attention3d(q, q, "auto", True, 3)
        o, l = torch.ops.cca.forward(q[:, :, 0], q[:, :, 0], v[:, :, 0])
        for call in (lambda: torch.ops.cca.forward3d(q, q, v, True, 3, "tc", True),
                     lambda: torch.ops.cca.backward3d(out, q, q, v, out, lse, True, 3, "tc"),
                     lambda: torch.ops.cca.attention3d_backward(attn, attn, q, q, "tc", True, 3, False),
                     lambda: torch.ops.cca.backward(o, q[:, :, 0], q[:, :, 0], v[:, :, 0], o, l, "tc")):
            with pytest.raises(RuntimeError, match="do not cover"):
                call()
