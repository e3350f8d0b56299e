"""CPU tests of float16 I/O: the C ABI accepts CCA_F16 where it accepts CCA_BF16, the Python layer routes torch.float16 to it,
and the f16 instantiations of the tensor-core kernels (ccnet_b200/csrc/cca_tc_f16.cu) compile as their bf16 counterparts do:
168 registers, no spills, asynchronous wgmmas, TMA stores / reduce-adds for the backward's outputs -- with f16 MMAs."""
import os
import re

import pytest
import torch

import ccnet_b200
from ccnet_b200 import build, capi
from ccnet_b200 import functional as F_
from test_bwd_kernel_outputs import _kernel_sass
from test_kernel_resources import _ptxas_report, _resources

F16_SRC = os.path.join(build.CSRC, "cca_tc_f16.cu")
SHAPES = [(8, 64, 512, 97, 97), (1, 64, 512, 193, 193), (2, 16, 64, 20, 30), (1, 8, 64, 32, 32)]


def test_f16_is_accepted_where_bf16_is():
    lib = capi.load()
    assert capi.CCA_F16 == 2
    for which in (capi.CCA_WS_FORWARD, capi.CCA_WS_BACKWARD):
        for shape in SHAPES:
            assert (lib.cca_b200_workspace_bytes(which, *shape, capi.CCA_F16)
                    == lib.cca_b200_workspace_bytes(which, *shape, capi.CCA_BF16) > 0), shape
            assert (lib.cca_b200_tc_supported(which, *shape, capi.CCA_F16)
                    == lib.cca_b200_tc_supported(which, *shape, capi.CCA_BF16)), shape
    # dtype 2 passes the dimension check and fails on the null pointers; 3 and above are still rejected
    rc = lib.cca_b200_forward(None, None, None, None, None, None, 0, 1, 8, 64, 4, 4, capi.CCA_F16, 0, None)
    assert rc == -1 and b"null" in lib.cca_b200_last_error()
    rc = lib.cca_b200_backward(*([None] * 10), 0, 1, 8, 64, 4, 4, capi.CCA_F16, 0, None)
    assert rc == -1 and b"null" in lib.cca_b200_last_error()
    for bad in (3, 7):
        rc = lib.cca_b200_forward(None, None, None, None, None, None, 0, 1, 8, 64, 4, 4, bad, 0, None)
        assert rc == -1 and b"dtype" in lib.cca_b200_last_error()
        assert lib.cca_b200_tc_supported(capi.CCA_WS_FORWARD, 8, 64, 512, 97, 97, bad) == 0
    # (the tensor-core predicate also needs the driver's tensor-map encoder, so it answers 0 on a machine without one)
    rc = lib.cca_b200_forward_host(None, None, None, None, None, 1, 8, 64, 4, 4, capi.CCA_F16, 0)
    assert rc == -1 and b"null" in lib.cca_b200_last_error()


def test_python_layer_maps_float16():
    assert F_._DTYPES[torch.float16] == capi.CCA_F16
    for shape in SHAPES:
        assert F_.tc_eligible(*shape, torch.float16) == F_.tc_eligible(*shape, torch.bfloat16), shape
    assert not F_.tc_eligible(1, 8, 64, 32, 32, torch.float16)
    # lines longer than one tile: both 16-bit types run on the fp32 kernels and round once (unless the native switch is set)
    for dt in (torch.float16, torch.bfloat16):
        assert F_._upcast(dt, 97, 193, False) and not F_._upcast(dt, 97, 97, False)
    assert not F_._upcast(torch.float32, 193, 193, False)
    with pytest.raises(RuntimeError, match="CUDA"):
        ccnet_b200.cca_forward(*(torch.randn(1, c, 4, 4, dtype=torch.float16) for c in (8, 8, 64)))


def fake_outputs(dtype):
    """torch.ops.cca.forward / backward under FakeTensorMode at a tensor-core shape: [(dtype, channels-last?) of out, dq, dk, dv]"""
    from torch._subclasses.fake_tensor import FakeTensorMode
    with FakeTensorMode():
        q = torch.empty(2, 64, 20, 30, device="cuda", dtype=dtype)
        v = torch.empty(2, 512, 20, 30, device="cuda", dtype=dtype)
        out, lse = torch.ops.cca.forward(q, q, v)
        assert lse.dtype == torch.float32 and lse.shape == (2, 20, 30)
        grads = torch.ops.cca.backward(out, q, q, v, out, lse)
        assert [g.shape for g in grads] == [q.shape, q.shape, v.shape]
        return [(t.dtype, t.is_contiguous(memory_format=torch.channels_last)) for t in (out, *grads)]


def test_fake_implementations_treat_fp16_as_bf16():
    """fp16 outputs in the memory format of bf16 ones: channels-last wherever the tensor-core kernels run (on an H100;
    tests/test_gpu_f16.py checks that case), NCHW where they do not."""
    assert fake_outputs(torch.float16) == [(torch.float16, cl) for _, cl in fake_outputs(torch.bfloat16)]


def test_f16_kernels_compile_like_the_bf16_kernels(tmp_path):
    report = _ptxas_report(F16_SRC, tmp_path)
    for kernel in ("cca_tc_stats_kernel", "cca_tc_fwd_kernel", "cca_tc_bwd_kernel"):
        res = _resources(report, kernel)
        assert len(res) == 2 and all("6__half" in n for n in res), res         # LK = 80, 112; f16 only
        assert all(v[:2] == (0, 0) for v in res.values()), res
        if kernel != "cca_tc_stats_kernel":
            assert all(v[2] == 168 for v in res.values()), res
    serialised = [line for line in report.splitlines() if "serialized" in line or re.search(r"\(C751[0-8]\)", line)]
    assert not serialised, "\n".join(serialised)

    sass = _kernel_sass(str(tmp_path / "k.o"), "_kernelILi")     # the six templates (not the prep kernel)
    assert len(sass) == 6, list(sass)
    for name, text in sass.items():
        mma = re.findall(r"HGMMA\.64x(\d+)x16\.(\S+)", text)
        real = [m for m in mma if m[0] != "8"]        # (64x8x16 with RZ operands: the compiler's own wait instruction)
        assert real, f"no HGMMA in {name}"
        assert all(ty == "F32" for _, ty in real), f"not the f16 form of HGMMA in {name}: {set(real)}"
    for name, text in sass.items():
        if "cca_tc_bwd_kernel" not in name:
            continue
        for op in ("UTMASTG.4D", "UTMAREDG.4D.ADD"):
            assert op in text, f"no {op} in {name}"
        assert not re.search(r"ATOM\S*\.ADD\.F16x2|ATOMG\.E\.ADD\.F32x2|ATOMS\.CAST", text), name
