"""CPU tests of the deterministic mode (CCA_FLAG_DETERMINISTIC) on tiled lines: the partial-plane mapping of the planes-mode
kernels writes every (pixel, plane) pair exactly once, the workspace query adds the planes only where they are used, and the
planes-mode instantiations (cca_tc_det.cu) compile as the default ones do.

Plane of an item (cca_items.cuh, read through cca_b200_item_planes): out and dQ by (direction, key block) = part_index, dK
and dV by (direction, query tile) = qtile_part_index; rows first, then columns."""
import ctypes
import os
import re

import numpy as np
import pytest

from ccnet_b200 import build, capi
from test_bwd_kernel_outputs import _kernel_sass
from test_items_host import _item, _space
from test_kernel_resources import _ptxas_report, _resources

TILED = [(2, 113, 200), (1, 7, 225), (2, 129, 257), (1, 896, 3)]
DET_NHWC = capi.CCA_FLAG_DETERMINISTIC | capi.CCA_FLAG_NHWC


def _planes(B, H, W, idx, lagged):
    out = (ctypes.c_int * 2)()
    capi.load().cca_b200_item_planes(B, H, W, idx, lagged, out)
    return out[0], out[1]


@pytest.mark.parametrize("lagged", [0, 1])
@pytest.mark.parametrize("shape", TILED)
def test_planes_are_written_exactly_once(shape, lagged):
    B, H, W = shape
    sp = _space(B, H, W)
    ntr, ntc = sp["ntr"], sp["ntc"]
    nparts = ntr + ntc
    assert nparts > 2
    by_key = np.zeros((nparts, B, H, W), np.int32)      # out, dQ: rows of the query tile, plane of the key block
    by_query = np.zeros((nparts, B, H, W), np.int32)    # dK, dV: rows of the key block, plane of the query tile
    for idx in range(sp["total"]):
        it = _item(B, H, W, idx, lagged)
        b, line = it["b"], it["line"]
        kplane, qplane = _planes(B, H, W, idx, lagged)
        # the same (direction, block) planes of the partial log-sum-exp: rows first, then columns
        assert kplane == (ntr + it["ik"] if it["col"] else it["ik"]) and qplane == (ntr + it["iq"] if it["col"] else it["iq"])
        qs, ks = slice(it["q0"], it["q0"] + it["lq"]), slice(it["k0"], it["k0"] + it["lk"])
        if it["col"]:
            by_key[kplane, b, qs, line] += 1
            by_query[qplane, b, ks, line] += 1
        else:
            by_key[kplane, b, line, qs] += 1
            by_query[qplane, b, line, ks] += 1
    assert (by_key == 1).all() and (by_query == 1).all()


def _ws(which, B, Cq, C, H, W, dtype, flags):
    lib = capi.load()
    return lib.cca_b200_workspace_bytes_ex(which, B, Cq, C, H, W, dtype, flags), lib.cca_b200_workspace_bytes(which, B, Cq, C, H, W, dtype)


@pytest.mark.parametrize("shape", [(2, 64, 128, 113, 200), (1, 16, 64, 7, 225), (8, 64, 512, 128, 128)])
def test_workspace_holds_the_planes(shape):
    B, Cq, C, H, W = shape
    nparts = -(-H // 112) + -(-W // 112)
    planes = {capi.CCA_WS_FORWARD: nparts * B * H * W * C * 4, capi.CCA_WS_BACKWARD: nparts * B * H * W * (2 * Cq + C) * 4}
    for which, need in planes.items():
        ex, plain = _ws(which, B, Cq, C, H, W, capi.CCA_F32, DET_NHWC)
        assert ex >= plain + need, (which, ex, plain, need)
        # no planes without the flag, without channels-last, or for 16-bit I/O (refused on such lines)
        assert _ws(which, B, Cq, C, H, W, capi.CCA_F32, capi.CCA_FLAG_NHWC)[0] == plain
        assert _ws(which, B, Cq, C, H, W, capi.CCA_F32, capi.CCA_FLAG_DETERMINISTIC)[0] == plain
        assert _ws(which, B, Cq, C, H, W, capi.CCA_BF16, DET_NHWC)[0] == plain


@pytest.mark.parametrize("shape", [(8, 64, 512, 97, 97), (1, 16, 64, 112, 112), (1, 8, 64, 200, 7), (1, 16, 64, 897, 3)])
def test_workspace_unchanged_on_one_tile_and_generic_shapes(shape):
    """one tile per line (already deterministic) and shapes only the generic kernels take (Cq = 8, a line of 897)"""
    for which in (capi.CCA_WS_FORWARD, capi.CCA_WS_BACKWARD):
        ex, plain = _ws(which, *shape, capi.CCA_F32, DET_NHWC)
        assert ex == plain


def test_wgrad_workspace_query():
    lib = capi.load()
    assert lib.cca_b200_qkv_wgrad_workspace_bytes(512, 64) >= (2 * 64 + 512) * 512 * 4       # at least one split
    assert lib.cca_b200_qkv_wgrad_workspace_bytes(100, 64) == 0                              # not covered


def test_planes_kernels_compile_like_the_default_ones(tmp_path):
    """the fp32 planes-mode forward and backward: no spills, 168 registers, asynchronous wgmma; they only STORE their tiles"""
    report = _ptxas_report(os.path.join(build.CSRC, "cca_tc_det.cu"), tmp_path)
    for kernel in ("cca_tc_fwd_kernel", "cca_tc_bwd_kernel"):
        res = _resources(report, kernel)
        assert len(res) == 2 and all("Lb1E" in n for n in res), res         # LK = 80, 112; fp32 planes mode only
        assert all(v == (0, 0, 168) for v in res.values()), res
    serialised = [line for line in report.splitlines() if "serialized" in line or re.search(r"\(C751[0-8]\)", line)]
    assert not serialised, "\n".join(serialised)
    sass = _kernel_sass(str(tmp_path / "k.o"), "_kernelILi")
    assert len(sass) == 4, list(sass)
    for name, text in sass.items():
        assert "UTMASTG.4D" in text, name
        assert "UTMAREDG" not in text, f"reduce-add in {name}"
