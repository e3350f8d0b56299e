"""Per-kernel SASS comparison of two builds of the library: which kernels compile to the same instructions.

    python tools/sass_compare.py OLD_LIBDIR NEW_LIBDIR [object ...]

Each LIBDIR is a build directory of ccnet_b200/build.py (CCA_B200_LIBDIR=... python -m ccnet_b200.build), holding one .o per
source.  Kernels are matched by mangled name after the per-build hash of anonymous namespaces is removed, and compared
instruction by instruction (column padding ignored).  ptxas is not bit-reproducible for every kernel: compiling the same
source twice can already differ (cca_simt.cu's line kernels do), so a difference means something only where two builds of
the parent agree.
"""
from __future__ import annotations

import os
import re
import subprocess
import sys


def kernels(obj: str) -> dict:
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    out = re.sub(r"_cu_[0-9a-f]{8}(_\d{4})?", "_cu_X", out)
    res, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            res[name] = []
        elif name and line.strip() and "identifier" not in line:
            res[name].append(" ".join(line.split()))
    return res


def main(old: str, new: str, objs) -> int:
    objs = objs or sorted(f for f in os.listdir(old) if f.endswith(".o"))
    same_all = True
    for o in objs:
        a, b = kernels(os.path.join(old, o)), kernels(os.path.join(new, o))
        same = [n for n in a if b.get(n) == a[n]]
        differ = [n for n in a if n not in same]
        same_all &= not differ
        print(f"{o}: {len(a)} kernels before, {len(same)} identical, {len(differ)} different, {len([n for n in b if n not in a])} new")
        for n in differ:
            print("   differs:", n)
    return 0 if same_all else 1


if __name__ == "__main__":
    sys.exit(main(sys.argv[1], sys.argv[2], sys.argv[3:]))
