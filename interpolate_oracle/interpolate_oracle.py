"""ctypes loader for the interpolation CPU oracle (interpolate_oracle/libinterpolate_oracle.so).  TEST INFRASTRUCTURE
ONLY.

May be imported only by tests/ and scripts/.  See interpolate_oracle.h for the rule.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libinterpolate_oracle.so")

LAYOUTS = {"f32": 0, "f16": 1, "cov": 2}

_lib = None


def build() -> None:
    subprocess.run(["make", "-C", _HERE, "-s"], check=True)


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        lib = C.CDLL(LIB_PATH)
        lib.orc_interp_factor.argtypes = [C.c_float, C.c_float, C.c_float, C.POINTER(C.c_float)]
        lib.orc_interp_factor.restype = C.c_int
        lib.orc_interp.argtypes = [C.c_uint32, C.c_int, C.c_float, C.c_void_p * 4, C.c_void_p * 4, C.c_void_p * 4]
        lib.orc_interp.restype = None
        lib.orc_half_to_float.argtypes = [C.c_uint16]
        lib.orc_half_to_float.restype = C.c_float
        lib.orc_float_to_half.argtypes = [C.c_float]
        lib.orc_float_to_half.restype = C.c_uint16
        _lib = lib
    return _lib


def factor(time: float, time_start: float, time_stop: float) -> np.float32:
    """The factor t as f32; ValueError for the inputs libbgs refuses (not finite, or a NaN factor)."""
    t = C.c_float()
    if load().orc_interp_factor(C.c_float(time), C.c_float(time_start), C.c_float(time_stop), C.byref(t)) != 0:
        raise ValueError("interpolate: no factor")
    return np.frombuffer(bytes(t), np.float32)[0]


def _planes_ptrs(planes):
    arr = C.c_void_p * 4
    ptrs = [p.ctypes.data for p in planes] + [None] * (4 - len(planes))
    return arr(*ptrs)


def interpolate(layout: str, lhs, rhs, t) -> tuple[np.ndarray, ...]:
    """mix(lhs, rhs, t) of two clouds given as their upload planes (f32: pos_vis, sh, rot, scale_opacity; f16 and cov:
    pos_vis, sh_packed, second plane) -> the output planes in the same form."""
    f32 = layout == "f32"
    kinds = [np.float32] * 4 if f32 else [np.float32, np.uint32, np.uint32]
    L = [np.ascontiguousarray(a, k) for a, k in zip(lhs, kinds)]
    R = [np.ascontiguousarray(a, k) for a, k in zip(rhs, kinds)]
    n = len(L[0])
    assert all(len(a) == n for a in L + R)
    out = [np.empty_like(a) for a in L]
    load().orc_interp(n, LAYOUTS[layout], C.c_float(np.float32(t)), _planes_ptrs(L), _planes_ptrs(R), _planes_ptrs(out))
    return tuple(out)


def half_to_float(h: int) -> np.float32:
    return np.float32(load().orc_half_to_float(int(h)))


def float_to_half(f) -> int:
    return int(load().orc_float_to_half(C.c_float(np.float32(f))))
