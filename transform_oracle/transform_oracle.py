"""ctypes loader for the transform CPU oracle (transform_oracle/libtransform_oracle.so).  TEST INFRASTRUCTURE ONLY.

May be imported only by tests/ and scripts/.  See transform_oracle.h for the rule.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtransform_oracle.so")

LAYOUTS = {"f32": 0, "f16": 1, "cov": 2}
SH_WIDTHS = (4, 12, 28, 48)

_lib = None


def build() -> None:
    subprocess.run(["make", "-C", _HERE, "-s"], check=True)


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        lib = C.CDLL(LIB_PATH)
        lib.orc_xf_sh_matrix.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        lib.orc_xf_sh_matrix.restype = None
        lib.orc_xf_params.argtypes = [C.c_void_p] + [C.c_void_p] * 5
        lib.orc_xf_params.restype = C.c_int
        lib.orc_xf_apply.argtypes = [C.c_uint32, C.c_int, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p * 4, C.c_void_p]
        lib.orc_xf_apply.restype = C.c_int
        _lib = lib
    return _lib


def column_major(matrix) -> np.ndarray:
    """A 4x4 matrix (row, column) as the 16 column-major f32 the call takes."""
    return np.ascontiguousarray(np.asarray(matrix, np.float32).T.reshape(16))


def sh_matrix(R, l: int) -> np.ndarray:
    """E_l = D_l^T, (2l+1, 2l+1) float64, for the rotation R (3x3), D_l defined by Y_l(R^T d) = D_l Y_l(d)."""
    R = np.ascontiguousarray(R, np.float64)
    m = 2 * l + 1
    E = np.empty((m, m), np.float64)
    load().orc_xf_sh_matrix(R.ctypes.data, l, E.ctypes.data)
    return E


def params(matrix):
    """(q_R (4,) f32 in w, x, y, z order, s f32, [E_1, E_2, E_3] f32) for a matrix the call accepts; None for one it
    refuses."""
    M = column_major(matrix)
    q, s = np.empty(4, np.float32), np.empty(1, np.float32)
    E = [np.empty((2 * l + 1, 2 * l + 1), np.float32) for l in (1, 2, 3)]
    if load().orc_xf_params(M.ctypes.data, q.ctypes.data, s.ctypes.data, *(e.ctypes.data for e in E)) != 0:
        return None
    return q, s[0], E


def accepts(matrix) -> bool:
    return load().orc_xf_params(column_major(matrix).ctypes.data, None, None, None, None, None) == 0


def transform(layout: str, degree: int, planes, matrix, selected: bool = False):
    """The transformed upload planes (f32: pos_vis, sh, rot, scale_opacity; f16 and cov: pos_vis, sh_packed, second
    plane) and, per SH lane, sum_j |E_ij c_j| (n, S_d) float64.  ValueError for a matrix the call refuses."""
    kinds = [np.float32] * 4 if layout == "f32" else [np.float32, np.uint32, np.uint32]
    out = [np.array(a, k, copy=True, order="C") for a, k in zip(planes, kinds)]
    n = len(out[0])
    bound = np.zeros((n, SH_WIDTHS[degree]), np.float64)
    ptrs = (C.c_void_p * 4)(*([a.ctypes.data for a in out] + [None] * (4 - len(out))))
    M = column_major(matrix)
    if load().orc_xf_apply(n, LAYOUTS[layout], degree, M.ctypes.data, 1 if selected else 0, ptrs, bound.ctypes.data) != 0:
        raise ValueError("transform: the matrix is refused")
    return tuple(out), bound
