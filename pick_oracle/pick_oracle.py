"""ctypes loader for bgs_render_entities_pick's oracle (pick_oracle/libpick_oracle.so).  TEST INFRASTRUCTURE ONLY.

May be imported only by tests/ and scripts/.  See pick_oracle.cpp for the rule.  `frame` is entity_oracle.frame's dict.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpick_oracle.so")

_lib = None


def build() -> None:
    subprocess.run(["make", "-C", _HERE, "-s"], check=True)


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        _lib = C.CDLL(LIB_PATH)
        _lib.po_pick.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32] + [C.c_void_p] * 6 + [C.c_double, C.c_double] + [C.c_void_p] * 6
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def pairs(frame: dict, kinds, W: int, H: int, coefs, scene=None) -> dict:
    """Every blending pair of every pixel: offsets ((H W + 1,) u64 into the pair arrays, pixel-major), rank, w (f64), bound
    (on the kernel's |w - w_f32|) and near_stop ((H, W) bool).  `kinds`: each rank's kind byte (0 quad-uv, 1 conic, | 4
    for the overlay); `coefs`: blend_cases.alpha_error_coefs' (c0, c1)."""
    n_vis = int(frame["n_vis"])
    recs = np.ascontiguousarray(frame["records"], np.float32)
    kinds = np.ascontiguousarray(kinds, np.uint8)
    assert kinds.shape == (n_vis,)
    rng = np.ascontiguousarray(frame["tile_ranges"], np.uint32)
    ent = np.ascontiguousarray(frame["tile_entries"], np.uint32)
    d = np.ascontiguousarray(frame["depths"], np.float32)
    sc = None if scene is None else np.ascontiguousarray(scene, np.float32)
    counts = np.zeros(W * H, np.uint32)
    head = [W, H, n_vis, _p(recs), _p(kinds), _p(rng), _p(ent), _p(d), _p(sc), float(coefs[0]), float(coefs[1])]
    rc = load().po_pick(*head, _p(counts), None, None, None, None, None)
    if rc != 0:
        raise ValueError("pick_oracle: surfel records are not restated")
    off = np.zeros(W * H + 1, np.uint64)
    np.cumsum(counts, out=off[1:])
    m = int(off[-1])
    rank, w, bound = np.empty(m, np.uint32), np.empty(m, np.float64), np.empty(m, np.float64)
    near = np.empty(W * H, np.uint8)
    assert load().po_pick(*head, _p(counts), _p(off), _p(rank), _p(w), _p(bound), _p(near)) == 0
    return dict(offsets=off, rank=rank, w=w, bound=bound, near_stop=near.reshape(H, W).astype(bool))
