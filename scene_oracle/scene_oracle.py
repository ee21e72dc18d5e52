"""ctypes loader for bgs_render_scene's oracle (scene_oracle/libscene_oracle.so).  TEST INFRASTRUCTURE ONLY.

May be imported only by tests/ and scripts/.  See scene_oracle.h for the rule.  `clouds`: a sequence of (cloud, uniform,
cov_pre): the cloud's planes as the oracle reads them (PlanarGaussian3d at SH degree 3; f16 clouds rounded, covariance
clouds decoded), its bgs_cloud_uniform (or orc_uniform), and whether its planes hold covariance records.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libscene_oracle.so")


class sor_cloud(C.Structure):
    _fields_ = [("n", C.c_uint32), ("cov_pre", C.c_uint32), ("pos_vis", C.c_void_p), ("sh", C.c_void_p), ("rot", C.c_void_p),
                ("scale_opacity", C.c_void_p), ("u", O.orc_uniform)]


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


def _clouds(clouds):
    """(ctypes array of sor_cloud, the arrays it points into: kept alive by the caller)"""
    keep, arr = [], (sor_cloud * len(clouds))()
    for j, (cloud, u, cov_pre) in enumerate(clouds):
        planes = [np.ascontiguousarray(a, np.float32) for a in
                  (cloud.position_visibility, cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity)]
        assert planes[1].shape[1] == 48, "the oracle reads SH degree 3 (pad lower degrees)"
        keep += planes
        arr[j] = sor_cloud(len(cloud), 1 if cov_pre else 0, *[p.ctypes.data for p in planes], O._conv(u, O.orc_uniform))
    return arr, keep


def sorted_entries(clouds, view, depth_bits: int = 32) -> np.ndarray:
    """(N, 2) uint32: the joint sorted entry list (key, global index)."""
    arr, keep = _clouds(clouds)
    n = sum(len(c) for c, _, _ in clouds)
    out = np.empty((n, 2), np.uint32)
    rc = load().sor_sorted_entries(C.c_uint32(len(clouds)), arr, C.byref(O._conv(view, O.orc_view)), C.c_uint32(depth_bits), _p(out))
    assert rc == 0, rc
    return out


def render_tiles(clouds, view, settings, want_image: bool = True, threads: int = 0):
    """-> dict(image, tile_ranges (T,2), tile_entries (I,), n_pairs, n_vis, rank_to_id, records), as oracle.render_tiles."""
    arr, keep = _clouds(clouds)
    v, s = O._conv(view, O.orc_view), O._conv(settings, O.orc_settings)
    W, H = int(v.viewport[2]), int(v.viewport[3])
    T = ((W + 15) // 16) * ((H + 15) // 16)
    head = (C.c_uint32(len(clouds)), arr, C.byref(v), C.byref(s))
    n_pairs, n_vis = C.c_uint64(), C.c_uint32()
    ranges = np.empty((T, 2), np.uint32)
    rc = load().sor_render_tiles(*head, None, _p(ranges), None, C.c_uint64(0), C.byref(n_pairs), C.byref(n_vis), None, None,
                                 C.c_int(threads))
    assert rc == 0, rc
    entries = np.empty(n_pairs.value, np.uint32)
    r2i = np.empty(n_vis.value, np.uint32)
    recs = np.zeros(n_vis.value, O.SPLAT_DTYPE)
    img = np.empty((H, W, 4), np.float32) if want_image else None
    rc = load().sor_render_tiles(*head, _p(img), _p(ranges), _p(entries), C.c_uint64(n_pairs.value), C.byref(n_pairs),
                                 C.byref(n_vis), _p(r2i), _p(recs), C.c_int(threads))
    assert rc == 0, rc
    return dict(image=img, tile_ranges=ranges, tile_entries=entries, n_pairs=n_pairs.value, n_vis=n_vis.value, rank_to_id=r2i,
                records=recs)


def render_ref(clouds, view, settings, dst: np.ndarray | None = None, threads: int = 0) -> np.ndarray:
    """ref_mode frame of the joint set over `dst` ((H, W, 4) premultiplied; None = opaque black)."""
    arr, keep = _clouds(clouds)
    v, s = O._conv(view, O.orc_view), O._conv(settings, O.orc_settings)
    W, H = int(v.viewport[2]), int(v.viewport[3])
    out = np.empty((H, W, 4), np.float32)
    if dst is not None:
        dst = np.ascontiguousarray(dst, np.float32)
        assert dst.shape == (H, W, 4)
    rc = load().sor_render_ref_over(C.c_uint32(len(clouds)), arr, C.byref(v), C.byref(s), _p(dst), _p(out), C.c_int(threads))
    assert rc == 0, rc
    return out
