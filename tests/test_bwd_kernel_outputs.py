"""CPU test: the backward attention kernel writes dQ, dK and dV with TMA, not with register atomics, and keeps its wgmmas async.

Each output tile of cca_tc_bwd_kernel is staged in shared memory and written by one thread with a TMA store (the producer
items of a sample) or a TMA reduce-add at L2 (all other items).  Per-thread global atomics on the outputs would sit on the
critical path of the chunk loop: every fp32 consumer thread used to issue 8 float2 atomics per 32-channel dV chunk, each
generic-address atomic with a shared-memory CAS fallback.  Only the u32 counter atomics and the 32-bit delta stores remain.
A spill, or an accumulator read inside another group's pipeline stage, would serialise the wgmmas (C7510-C7518); the
injected arrives of the S = Q K^T loop (C7519) are allowed.  Compiled as in tests/test_kernel_resources.py.
"""
import re
import subprocess

import pytest

from ccnet_b200 import build
from test_kernel_resources import BWD_SRC, _ptxas_report, _resources


def _kernel_sass(obj, kernel):
    """{function name: SASS text} of the functions whose name contains `kernel`"""
    cuobjdump = build._nvcc().replace("nvcc", "cuobjdump")
    out = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True)
    if out.returncode != 0:
        pytest.skip("cuobjdump unavailable: " + out.stderr[-200:])
    funcs, name = {}, None
    for line in out.stdout.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1) if kernel in m.group(1) else None
            if name:
                funcs[name] = []
            continue
        if name:
            funcs[name].append(line)
    return {k: "\n".join(v) for k, v in funcs.items()}


def test_backward_kernel_writes_outputs_with_tma(tmp_path):
    report = _ptxas_report(BWD_SRC, tmp_path)
    res = _resources(report, "cca_tc_bwd_kernel")
    # <LK = 80, 112> x <fp32, bf16>
    assert len(res) == 4, res
    assert all(v == (0, 0, 168) for v in res.values()), res
    serialised = [line for line in report.splitlines() if "serialized" in line or re.search(r"\(C751[0-8]\)", line)]
    assert not serialised, "\n".join(serialised)

    sass = _kernel_sass(str(tmp_path / "k.o"), "cca_tc_bwd_kernel")
    assert len(sass) == 4, list(sass)
    for name, text in sass.items():
        for op in ("ATOMG.E.ADD.F32x2", "ATOM.E.ADD.BF16x2", "ATOMS.CAST", "STG.E.64"):
            assert op not in text, f"{op} in {name}"
        for op in ("UTMASTG.4D", "UTMAREDG.4D.ADD"):
            assert op in text, f"no {op} in {name}"
        assert re.search(r"STG\.E [^\n]*", text), f"no delta store in {name}"
