"""ctypes loader for the SparseSelect and point-in-mesh CPU oracle (select_oracle/libselect_oracle.so).  TEST INFRASTRUCTURE ONLY.

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
        margs = [C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                 C.POINTER(C.c_uint32), C.c_int]
        for name in ("orc_select_in_mesh", "orc_select_in_mesh_grid"):
            getattr(lib, name).argtypes = margs
            getattr(lib, name).restype = C.c_int
        lib.orc_mesh_plan.argtypes = [C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32),
                                      C.POINTER(C.c_uint64)]
        lib.orc_mesh_plan.restype = C.c_int
        lib.orc_mesh_boxes.argtypes = [C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.orc_mesh_boxes.restype = C.c_int
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


def _mesh(vertices, indices):
    v = np.ascontiguousarray(vertices, np.float32).reshape(-1, 3)
    i = np.ascontiguousarray(indices, np.uint32).reshape(-1, 3)
    return v, i


def select_in_mesh(pos_vis: np.ndarray, vertices, indices, mesh_from_cloud=None, grid: bool = False, threads: int = 0):
    """-> (inside mask (n,) bool, inside count).  mesh_from_cloud: 4x4 numpy (M @ p), None = identity.
    grid=False: every (point, triangle) pair (the definition); True: libbgs's grid restated."""
    p = _pos(pos_vis)
    v, i = _mesh(vertices, indices)
    m = None if mesh_from_cloud is None else np.ascontiguousarray(np.asarray(mesh_from_cloud, np.float32).T)
    mask = np.zeros(len(p), np.uint8)
    inside = C.c_uint32()
    fn = load().orc_select_in_mesh_grid if grid else load().orc_select_in_mesh
    rc = fn(len(p), p.ctypes.data_as(C.c_void_p), len(v), v.ctypes.data_as(C.c_void_p), len(i), i.ctypes.data_as(C.c_void_p),
            None if m is None else m.ctypes.data_as(C.c_void_p), mask.ctypes.data_as(C.c_void_p), C.byref(inside), C.c_int(threads))
    if rc != 0:
        raise ValueError("indices must be < the vertex count")
    return mask.astype(bool), int(inside.value)


def mesh_plan(vertices, indices) -> dict:
    """The grid the kernel builds for this mesh: binned / global triangle counts, (ny, nz), level (-1: none), pairs."""
    v, i = _mesh(vertices, indices)
    counts = np.zeros(4, np.uint32)
    level, pairs = C.c_int32(), C.c_uint64()
    rc = load().orc_mesh_plan(len(v), v.ctypes.data_as(C.c_void_p), len(i), i.ctypes.data_as(C.c_void_p),
                              counts.ctypes.data_as(C.c_void_p), C.byref(level), C.byref(pairs))
    if rc != 0:
        raise ValueError("indices must be < the vertex count")
    return {"binned": int(counts[0]), "global": int(counts[1]), "ny": int(counts[2]), "nz": int(counts[3]),
            "level": int(level.value), "pairs": int(pairs.value)}


def mesh_boxes(vertices, indices):
    """-> (class (nt,) int32: 0 dropped, 1 binned, 2 global; boxes (nt, 4) f64 ylo, yhi, zlo, zhi, NaN unless binned)."""
    v, i = _mesh(vertices, indices)
    box = np.empty((len(i), 4), np.float64)
    cls = np.empty(len(i), np.int32)
    rc = load().orc_mesh_boxes(len(v), v.ctypes.data_as(C.c_void_p), len(i), i.ctypes.data_as(C.c_void_p),
                               box.ctypes.data_as(C.c_void_p), cls.ctypes.data_as(C.c_void_p))
    if rc != 0:
        raise ValueError("indices must be < the vertex count")
    return cls, box
