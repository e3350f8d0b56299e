"""Record the C ABI's workspace sizes over a grid of shapes, dtypes and flags into ``workspace_bytes.json``.

    python tests/golden/make_workspace_bytes.py              (uses the library CCA_B200_LIB or the in-tree build)

Callers allocate by these sizes, so they are part of the ABI: tests/test_host_surface.py checks every recorded query
against the library.  The queries need no device.  The grid covers both kernel families' workspaces: one-tile and tiled
lines, shapes only the generic kernels take (a 897-pixel line, Cq = 8, C = 100), H = 1 and W = 1, one and eight samples,
and T = 1, 4, 32 and 33 for the 3D op.
"""
import itertools
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from ccnet_b200 import capi  # noqa: E402

OUT = os.path.join(HERE, "workspace_bytes.json")
DTYPES = [capi.CCA_F32, capi.CCA_BF16, capi.CCA_F16]
NHWC, DET = capi.CCA_FLAG_NHWC, capi.CCA_FLAG_DETERMINISTIC
FLAGS = [0, NHWC, NHWC | DET, DET]
WHICH = [capi.CCA_WS_FORWARD, capi.CCA_WS_BACKWARD]
BATCH = [1, 8]
CHANNELS = [(64, 512), (8, 100)]                                         # (Cq, C)
SHAPES = [(97, 97), (193, 193), (113, 7), (7, 896), (897, 16), (1, 97), (97, 1), (1, 1)]
SHAPES3D = [(97, 97), (193, 193), (7, 896), (1, 1)]
TIMES = [1, 4, 32, 33]


def grid():
    """query name -> list of argument tuples"""
    return {
        "cca_b200_workspace_bytes": [(w, b, cq, c, h, wd, dt) for w, b, (cq, c), (h, wd), dt
                                     in itertools.product(WHICH, BATCH, CHANNELS, SHAPES, DTYPES)],
        "cca_b200_workspace_bytes_ex": [(w, b, cq, c, h, wd, dt, f) for w, b, (cq, c), (h, wd), dt, f
                                        in itertools.product(WHICH, BATCH, CHANNELS, SHAPES, DTYPES, FLAGS)],
        "cca_b200_attention_workspace_bytes": [(w, b, cq, h, wd, dt, f) for w, b, (cq, _), (h, wd), dt, f
                                               in itertools.product(WHICH, BATCH, CHANNELS, SHAPES, DTYPES, FLAGS)],
        "cca_b200_workspace_bytes3d": [(w, b, cq, c, t, h, wd, dt, f) for w, b, (cq, c), t, (h, wd), dt, f
                                       in itertools.product(WHICH, BATCH, CHANNELS, TIMES, SHAPES3D, DTYPES, FLAGS)],
    }


def main():
    lib = capi.load()
    rows = {name: [[*args, getattr(lib, name)(*args)] for args in cases] for name, cases in grid().items()}
    with open(OUT, "w") as f:          # one case per line: [arguments..., bytes]
        f.write("{\n" + ",\n".join(
            f' "{name}": [\n' + ",\n".join("  " + json.dumps(r) for r in rs) + "\n ]" for name, rs in rows.items()) + "\n}\n")
    print(OUT, sum(len(r) for r in rows.values()), "cases")


if __name__ == "__main__":
    main()
