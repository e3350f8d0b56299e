"""Build the C-ABI shared library ``ccnet_b200/lib/libcca_b200.so`` with nvcc for sm_90a.

In-tree build (the .so is git-ignored; build() recompiles it).
``python -m ccnet_b200.build [--force]``
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.environ.get("CCA_B200_LIBDIR") or os.path.join(HERE, "lib")      # (override: a second build flavour)
LIB = os.path.join(LIBDIR, "libcca_b200.so")
SOURCES = ["cca_capi.cu", "cca_simt.cu", "cca_simt_attn.cu", "cca_simt_3d.cu", "cca_tc_host.cu", "cca_tc_stats.cu", "cca_tc_fwd.cu", "cca_tc_bwd.cu", "cca_tc_f16.cu",
           "cca_tc_det.cu", "cca_tc_attn.cu", "cca_tc_time.cu", "cca_tc_attn3d.cu", "cca_simt_attn3d.cu", "cca_gemm.cu",
           "cca_tc_causal.cu", "cca_simt_causal.cu"]
HEADERS = ["cca_common.cuh", "cca_sm90.cuh", "cca_tc_common.cuh", "cca_items.cuh", "cca_tc_stats.cuh", "cca_tc_fwd.cuh",
           "cca_tc_bwd.cuh", "cca_tc_attn.cuh", "cca_tc_time.cuh", "cca_tc_attn3d.cuh", "../../include/cca_b200.h"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo", "--use_fast_math",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


DEBUG_FLAGS = ["-DCCA_SPIN_TRAP=1", "-DCCA_DEBUG_HOOKS"]   # bounded spins that trap + the cca_b200__set_* A/B hooks


def build(force: bool = False, verbose: bool = False, debug: bool | None = None) -> str:
    """Release build by default; ``debug=True`` / ``--debug`` / CCA_B200_DEBUG_BUILD=1 adds DEBUG_FLAGS.  The flavour is
    recorded in lib/flavour.txt; changing it rebuilds everything."""
    os.makedirs(LIBDIR, exist_ok=True)
    if debug is None:
        debug = bool(os.environ.get("CCA_B200_DEBUG_BUILD"))
    flavour_flags = DEBUG_FLAGS if debug else []
    stamp = os.path.join(LIBDIR, "flavour.txt")
    flavour = " ".join(flavour_flags) or "release"
    if not os.path.exists(stamp) or open(stamp).read() != flavour:
        force = True
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    objs = []
    nvcc = _nvcc()
    extra = (["-Xptxas", "-v"] if verbose else []) + flavour_flags
    procs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(LIBDIR, s.replace(".cu", ".o"))
        objs.append(obj)
        if force or _stale(obj, [src] + hdrs):
            cmd = [nvcc, *NVCC_FLAGS, *extra, "-c", src, "-o", obj]
            procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"--- nvcc failed for {s} ---\n{out}\n")
        elif verbose:
            sys.stderr.write(out)
    if failed:
        raise RuntimeError("nvcc compilation failed")
    if force or procs or _stale(LIB, objs):
        subprocess.check_call([nvcc, "-shared", "-o", LIB, *objs, "-lcudart"])
    with open(stamp, "w") as f:
        f.write(flavour)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, debug=True if "--debug" in sys.argv else None))
