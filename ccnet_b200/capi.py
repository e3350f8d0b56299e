"""ctypes binding of the C ABI in ``include/cca_b200.h`` (``ccnet_b200/lib/libcca_b200.so``).

The library is the product; this module only marshals pointers.  There is NO fallback: if the
shared library is missing or a call fails, a ``RuntimeError`` is raised.
"""
from __future__ import annotations

import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("CCA_B200_LIB") or os.path.join(_HERE, "lib", "libcca_b200.so")   # (override: another build flavour)

CCA_F32, CCA_BF16 = 0, 1
CCA_FLAG_AUTO, CCA_FLAG_FORCE_SIMT, CCA_FLAG_FORCE_TC, CCA_FLAG_NHWC = 0, 1, 2, 4
CCA_WS_FORWARD, CCA_WS_BACKWARD = 0, 1

# every symbol include/cca_b200.h declares: name -> (restype, argtypes)
_vp, _i, _u, _sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint, ctypes.c_size_t
SYMBOLS = {
    "cca_b200_version": (_i, []),
    "cca_b200_last_error": (ctypes.c_char_p, []),
    "cca_b200_strerror": (ctypes.c_char_p, [_i]),
    "cca_b200_device_ok": (_i, []),
    "cca_b200_launch_count": (ctypes.c_ulonglong, []),
    "cca_b200_tc_supported": (_i, [_i] * 7),
    "cca_b200_item_space": (None, [_i] * 3 + [ctypes.POINTER(_i)]),
    "cca_b200_decode_item": (None, [_i] * 5 + [ctypes.POINTER(_i)]),
    "cca_b200_workspace_bytes": (_sz, [_i] * 7),
    "cca_b200_qkv_supported": (_i, [_i, _i]),
    "cca_b200_qkv_workspace_bytes": (_sz, [_i, _i]),
    "cca_b200_qkv_project": (_i, [_vp] * 11 + [_sz, ctypes.c_longlong, _i, _i, _vp]),
    "cca_b200_qkv_project_dgrad": (_i, [_vp] * 9 + [_sz, ctypes.c_longlong, _i, _i, _i, _vp]),
    "cca_b200_qkv_wgrad_supported": (_i, [_i, _i]),
    "cca_b200_qkv_project_wgrad": (_i, [_vp] * 9 + [ctypes.c_longlong, _i, _i, _vp]),
    "cca_b200_forward": (_i, [_vp] * 6 + [_sz] + [_i] * 6 + [_u, _vp]),
    "cca_b200_backward": (_i, [_vp] * 10 + [_sz] + [_i] * 6 + [_u, _vp]),
    "cca_b200_forward_host": (_i, [_vp] * 5 + [_i] * 6 + [_u]),
    "cca_b200_backward_host": (_i, [_vp] * 9 + [_i] * 6 + [_u]),
}

_lib = None
_lock = threading.Lock()


def load() -> ctypes.CDLL:
    """Load the shared library (once).  Raises RuntimeError if it has not been built."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise RuntimeError(
                        f"{LIB_PATH} not found: build it with `python -m ccnet_b200.build` "
                        "(ccnet_b200 has no CPU or PyTorch fallback)")
                lib = ctypes.CDLL(LIB_PATH)
                for name, (res, args) in SYMBOLS.items():
                    fn = getattr(lib, name)
                    fn.restype, fn.argtypes = res, args
                _lib = lib
    return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        lib = load()
        raise RuntimeError(f"{what} failed: {lib.cca_b200_strerror(rc).decode()} "
                           f"({lib.cca_b200_last_error().decode()})")


def launch_count() -> int:
    return int(load().cca_b200_launch_count())
