"""CPU test: the backward attention kernel compiles for sm_90a without register spills.

Every instantiation of cca_tc_bwd_kernel keeps its wgmma accumulators (dP, dV, dQ, dK) in registers; a spill puts local-memory
traffic into the chunk loop and makes ptxas serialise the kernel's wgmmas.  The file is compiled with the flags of
ccnet_b200/build.py plus ``-Xptxas -v`` and the spill counts ptxas reports are checked, as well as the launch register count
the setmaxnreg split of the warpgroups is sized for (cca_tc_common.cuh: 384 threads x 168 registers).
"""
import os
import re
import subprocess

import pytest

from ccnet_b200 import build

BWD_SRC = os.path.join(build.CSRC, "cca_tc_bwd.cu")


def _ptxas_report(src, tmp_path):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    out = subprocess.run([nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "k.o")],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    return out.stdout + out.stderr


def _resources(report, kernel):
    """{mangled instantiation name: (spill store bytes, spill load bytes, registers)} of the kernels whose name contains `kernel`"""
    res, name, spills = {}, None, None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name = m.group(1) if kernel in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            spills = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers", line)
        if m and name and spills:
            res[name] = spills + (int(m.group(1)),)
            name, spills = None, None
    return res


def test_backward_kernel_has_no_register_spills(tmp_path):
    res = _resources(_ptxas_report(BWD_SRC, tmp_path), "cca_tc_bwd_kernel")
    # <LK = 80, 112> x <fp32, bf16>
    assert len(res) == 4, res
    assert all(v == (0, 0, 168) for v in res.values()), res
