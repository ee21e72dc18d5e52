"""ctypes loader for bgs_render_entities' oracle (entity_oracle/libentity_oracle.so).  TEST INFRASTRUCTURE ONLY.

May be imported only by tests/ and scripts/.  See entity_oracle.h for the rule.  `clouds`: scene4d_oracle's entries,
(cloud, uniform, cov_pre) or (cloud4d, uniform, (time_start, time_stop)); `settings`: one bgs_settings (or orc_settings)
per cloud, and `num_classes` one count per cloud.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import oracle as O
from scene4d_oracle import scene4d_oracle as S4O
from temporal_oracle import temporal_oracle as T

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libentity_oracle.so")

_lib = None


def build() -> None:
    subprocess.run(["make", "-C", _HERE, "-s"], check=True)


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        _lib = C.CDLL(LIB_PATH)
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def frame(clouds, view, settings, num_classes=None, extras=None, scene=None, want_image: bool = True, threads: int = 0) -> dict:
    """-> s4o_frame's dict (sorted, records, rank_to_id, depths, tile_ranges, tile_entries, n_vis, n_pairs, image)."""
    arr, keep = S4O._clouds(clouds)
    k = len(clouds)
    sa = (O.orc_settings * k)(*[O._conv(s, O.orc_settings) for s in settings])
    nc = np.ascontiguousarray(num_classes if num_classes is not None else [1] * k, np.uint32)
    v = O._conv(view, O.orc_view)
    W, H = int(v.viewport[2]), int(v.viewport[3])
    nt = ((W + 15) // 16) * ((H + 15) // 16)
    ex = T.temporal(0.0, 1.0, extras)
    pitch = 0
    if scene is not None:
        scene = np.ascontiguousarray(scene, np.float32)
        pitch = scene.shape[1] * 4
    nv, npairs = C.c_uint32(), C.c_uint64()
    head = [C.c_uint32(k), arr, C.byref(v), sa, _p(nc), C.byref(ex), _p(scene), C.c_uint64(pitch), C.byref(nv), C.byref(npairs)]
    rc = load().eo_frame(*head, *([None] * 6), None, C.c_uint64(0), None, C.c_int(threads))
    assert rc == 0, rc
    n = sum(len(c) for c, _, _ in clouds)
    out = dict(sorted=np.empty((n, 2), np.uint32), records=np.empty((nv.value, 12), np.float32),
               rank_to_id=np.empty(nv.value, np.uint32), depths=np.empty(nv.value, np.float32),
               tile_ranges=np.empty((nt, 2), np.uint32), tile_entries=np.empty(npairs.value, np.uint32),
               image=np.empty((H, W, 4), np.float32) if want_image else None)
    assert load().eo_frame(*head, _p(out["sorted"]), _p(out["records"]), _p(out["rank_to_id"]), _p(out["depths"]),
                           _p(out["tile_ranges"]), _p(out["tile_entries"]), C.c_uint64(npairs.value), _p(out["image"]),
                           C.c_int(threads)) == 0
    out["n_vis"], out["n_pairs"] = nv.value, npairs.value
    return out
