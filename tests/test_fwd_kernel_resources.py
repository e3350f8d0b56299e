"""CPU test: the forward values kernel compiles for sm_90a without spills and without serialised wgmmas.

The chunk loop of cca_tc_fwd_kernel runs chunk n's O = P V group while the other O accumulator is staged for its TMA store
and chunk n + 1 is converted.  That overlap only exists if ptxas keeps the wgmmas asynchronous: a spill, or an accumulator
read inside another group's pipeline stage (C7514) or a wait ptxas has to insert in a divergent path (C7518), makes it wait
for every wgmma on its own (C7512 and relatives: "wgmma.mma_async instructions are serialized").  The injected arrives of
the S = Q K^T loop (C7519) do not serialise and are allowed.  Compiled as in tests/test_kernel_resources.py.
"""
import os
import re

from ccnet_b200 import build
from test_kernel_resources import _ptxas_report, _resources

FWD_SRC = os.path.join(build.CSRC, "cca_tc_fwd.cu")


def test_forward_kernel_has_no_spills_and_no_serialised_wgmma(tmp_path):
    report = _ptxas_report(FWD_SRC, tmp_path)
    res = _resources(report, "cca_tc_fwd_kernel")
    # <LK = 80, 112> x <fp32, bf16>
    assert len(res) == 4, res
    assert all(v == (0, 0, 168) for v in res.values()), res
    serialised = [line for line in report.splitlines() if "serialized" in line or re.search(r"\(C751[0-8]\)", line)]
    assert not serialised, "\n".join(serialised)
