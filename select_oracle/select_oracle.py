"""ctypes loader for the SparseSelect CPU oracle (select_oracle/libselect_oracle.so).  TEST INFRASTRUCTURE ONLY.

May be imported only by tests/ and scripts/.  See select_oracle.h for the selection rule and its parity status.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libselect_oracle.so")

_lib = None


def build() -> None:
    subprocess.run(["make", "-C", _HERE, "-s"], check=True)


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        lib = C.CDLL(LIB_PATH)
        args = [C.c_uint32, C.c_void_p, C.c_float, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32), C.c_int]
        for name in ("orc_select_sparse", "orc_select_sparse_grid"):
            getattr(lib, name).argtypes = args
            getattr(lib, name).restype = C.c_int
        lib.orc_select_buckets.argtypes = [C.c_uint32, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p]
        lib.orc_select_buckets.restype = C.c_uint32
        _lib = lib
    return _lib


def _pos(pos_vis: np.ndarray) -> np.ndarray:
    a = np.ascontiguousarray(pos_vis, np.float32)
    assert a.ndim == 2 and a.shape[1] == 4
    return a


def select_sparse(pos_vis: np.ndarray, radius: float, threshold: int, grid: bool = False, threads: int = 0):
    """-> (mask (n,) bool, selected count).  grid=False: brute force (the definition); True: the hashed grid."""
    p = _pos(pos_vis)
    n = len(p)
    mask = np.zeros(n, np.uint8)
    sel = C.c_uint32()
    fn = load().orc_select_sparse_grid if grid else load().orc_select_sparse
    rc = fn(n, p.ctypes.data_as(C.c_void_p), C.c_float(radius), C.c_uint32(threshold), mask.ctypes.data_as(C.c_void_p),
            C.byref(sel), C.c_int(threads))
    if rc != 0:
        raise ValueError(f"radius {radius!r} must be finite and >= 0")
    return mask.astype(bool), int(sel.value)


def buckets(pos_vis: np.ndarray, radius: float):
    """-> (bucket (n,) u32 -- n_buckets for a non-finite position --, cells (n, 3) i64, n_buckets)."""
    p = _pos(pos_vis)
    n = len(p)
    b = np.empty(n, np.uint32)
    cells = np.empty((n, 3), np.int64)
    nb = load().orc_select_buckets(n, p.ctypes.data_as(C.c_void_p), C.c_float(radius), b.ctypes.data_as(C.c_void_p),
                                   cells.ctypes.data_as(C.c_void_p))
    return b, cells, int(nb)
