"""ctypes loader for bgs_render_scene_4d's oracle (scene4d_oracle/libscene4d_oracle.so).  TEST INFRASTRUCTURE ONLY.

May be imported only by tests/ and scripts/.  See scene4d_oracle.h for the rule.  `clouds`: a sequence of entries,
either (cloud, uniform, cov_pre) for a 3D cloud as scene_oracle/ takes it (PlanarGaussian3d at SH degree 3, f16 clouds
rounded, covariance clouds decoded), or (cloud4d, uniform, (time_start, time_stop)) for a PlanarGaussian4d, whose time
is uniform.time.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import oracle as O
from temporal_oracle import temporal_oracle as T

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libscene4d_oracle.so")


class s4o_cloud(C.Structure):
    _fields_ = [("n", C.c_uint32), ("kind", C.c_uint32), ("cov_pre", C.c_uint32), ("pos_vis", C.c_void_p), ("sh", C.c_void_p),
                ("rot", C.c_void_p), ("scale_opacity", C.c_void_p), ("tt", C.c_void_p), ("u", O.orc_uniform),
                ("time_start", C.c_float), ("time_stop", C.c_float)]


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


def is_4d(cloud) -> bool:
    return hasattr(cloud, "timestamp_timescale")


def _clouds(clouds):
    """(ctypes array of s4o_cloud, the arrays it points into: kept alive by the caller)"""
    keep, arr = [], (s4o_cloud * len(clouds))()
    for j, (cloud, u, extra) in enumerate(clouds):
        if is_4d(cloud):
            planes = [np.ascontiguousarray(a, np.float32) for a in cloud.planes()]   # pos, sh144, rot8, so, tt
            keep += planes
            ts, te = extra
            arr[j] = s4o_cloud(len(cloud), 1, 0, *[p.ctypes.data for p in planes], O._conv(u, O.orc_uniform), float(ts), float(te))
        else:
            planes = [np.ascontiguousarray(a, np.float32) for a in
                      (cloud.position_visibility, cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity)]
            assert planes[1].shape[1] == 48, "the oracle reads SH degree 3 (pad lower degrees)"
            keep += planes
            arr[j] = s4o_cloud(len(cloud), 0, 1 if extra else 0, *[p.ctypes.data for p in planes], None, O._conv(u, O.orc_uniform),
                               0.0, 1.0)
    return arr, keep


def frame(clouds, view, settings, extras=None, scene=None, want_image: bool = True, threads: int = 0) -> dict:
    """-> dict(sorted (N, 2), records (n_vis, 12) in bgs_debug_projected's layout by rank, rank_to_id, depths, tile_ranges
    (T, 2), tile_entries, n_vis, n_pairs, image (H, W, 4) or None)."""
    arr, keep = _clouds(clouds)
    v, s = O._conv(view, O.orc_view), O._conv(settings, O.orc_settings)
    W, H = int(v.viewport[2]), int(v.viewport[3])
    nt = ((W + 15) // 16) * ((H + 15) // 16)
    ex = T.temporal(0.0, 1.0, extras)
    pitch = 0
    if scene is not None:
        scene = np.ascontiguousarray(scene, np.float32)
        pitch = scene.shape[1] * 4
    nv, npairs = C.c_uint32(), C.c_uint64()
    head = [C.c_uint32(len(clouds)), arr, C.byref(v), C.byref(s), C.byref(ex), _p(scene), C.c_uint64(pitch), C.byref(nv),
            C.byref(npairs)]
    assert load().s4o_frame(*head, *([None] * 6), None, C.c_uint64(0), None, C.c_int(threads)) == 0
    n = sum(len(c) for c, _, _ in clouds)
    out = dict(sorted=np.empty((n, 2), np.uint32), records=np.empty((nv.value, 12), np.float32),
               rank_to_id=np.empty(nv.value, np.uint32), depths=np.empty(nv.value, np.float32),
               tile_ranges=np.empty((nt, 2), np.uint32), tile_entries=np.empty(npairs.value, np.uint32),
               image=np.empty((H, W, 4), np.float32) if want_image else None)
    assert load().s4o_frame(*head, _p(out["sorted"]), _p(out["records"]), _p(out["rank_to_id"]), _p(out["depths"]),
                            _p(out["tile_ranges"]), _p(out["tile_entries"]), C.c_uint64(npairs.value), _p(out["image"]),
                            C.c_int(threads)) == 0
    out["n_vis"], out["n_pairs"] = nv.value, npairs.value
    return out
