"""ctypes loader for the depth-tested frame's oracle (depth_oracle/libdepth_oracle.so).  TEST INFRASTRUCTURE ONLY.

May be imported only by tests/ and scripts/.  See depth_oracle.h for the rule.  `scene`: an (H, W) float32 array, or an
(H, P) one of which the first W columns are the frame's (a padded pitch); None = no depth test.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdepth_oracle.so")

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


def _scene(scene, W: int, H: int):
    if scene is None:
        return None, 0
    scene = np.ascontiguousarray(scene, np.float32)
    assert scene.ndim == 2 and scene.shape[0] == H and scene.shape[1] >= W, scene.shape
    return scene, scene.strides[0]


def _cloud_args(cloud, view, uniform, settings):
    v, u, s = O._conv(view, O.orc_view), O._conv(uniform, O.orc_uniform), O._conv(settings, O.orc_settings)
    args = (C.c_uint32(len(cloud)), _p(cloud.position_visibility), _p(cloud.spherical_harmonic), _p(cloud.rotation),
            _p(cloud.scale_opacity), C.byref(v), C.byref(u), C.byref(s))
    return v, args


def splat_depth(pos_vis: np.ndarray, view, uniform, ids: np.ndarray) -> np.ndarray:
    """d of gaussians `ids` (include/bgs.h, bgs_render_depth_test)."""
    ids = np.ascontiguousarray(ids, np.uint32)
    pos_vis = np.ascontiguousarray(pos_vis, np.float32)
    out = np.empty(len(ids), np.float32)
    v, u = O._conv(view, O.orc_view), O._conv(uniform, O.orc_uniform)
    rc = load().dor_splat_depth(C.c_uint32(len(pos_vis)), _p(pos_vis), C.byref(v), C.byref(u), C.c_uint32(len(ids)), _p(ids),
                                _p(out))
    assert rc == 0, rc
    return out


def render_ref(cloud, view, uniform, settings, scene=None, dst: np.ndarray | None = None, threads: int = 0) -> np.ndarray:
    """ref_mode frame with the per-fragment depth test, back to front (over `dst`, None = opaque black)."""
    v, args = _cloud_args(cloud, view, uniform, settings)
    W, H = int(v.viewport[2]), int(v.viewport[3])
    z, pitch = _scene(scene, W, H)
    out = np.empty((H, W, 4), np.float32)
    if dst is not None:
        dst = np.ascontiguousarray(dst, np.float32)
    rc = load().dor_render_ref_over(*args, _p(dst), _p(z), C.c_uint64(pitch), _p(out), C.c_int(threads))
    assert rc == 0, rc
    return out


def render_tiles(cloud, view, uniform, settings, scene=None, threads: int = 0) -> np.ndarray:
    """tile_mode frame (over opaque black) with the depth test."""
    v, args = _cloud_args(cloud, view, uniform, settings)
    W, H = int(v.viewport[2]), int(v.viewport[3])
    z, pitch = _scene(scene, W, H)
    out = np.empty((H, W, 4), np.float32)
    rc = load().dor_render_tiles(*args, _p(z), C.c_uint64(pitch), _p(out), C.c_int(threads))
    assert rc == 0, rc
    return out


def blend_trace(cloud, view, uniform, settings, scene=None, threads: int = 0) -> np.ndarray:
    """(H, W) oracle.TRACE_DTYPE of the depth-tested tile walk."""
    v, args = _cloud_args(cloud, view, uniform, settings)
    W, H = int(v.viewport[2]), int(v.viewport[3])
    z, pitch = _scene(scene, W, H)
    out = np.zeros((H, W), O.TRACE_DTYPE)
    rc = load().dor_blend_trace(*args, _p(z), C.c_uint64(pitch), _p(out), C.c_int(threads))
    assert rc == 0, rc
    return out


def coverage_probe(splats: np.ndarray, settings, pixel_xy: np.ndarray, splat_d=None, scene_d=None) -> np.ndarray:
    """oracle.coverage_probe with the test: pair j is covered only if also splat_d[j] >= scene_d[j]."""
    splats = np.ascontiguousarray(splats, O.SPLAT_DTYPE)
    xy = np.ascontiguousarray(pixel_xy, np.float32).reshape(len(splats), 2)
    out = np.zeros(len(splats), O.PROBE_DTYPE)
    s = O._conv(settings, O.orc_settings)
    sd = None if splat_d is None else np.ascontiguousarray(splat_d, np.float32)
    zd = None if scene_d is None else np.ascontiguousarray(scene_d, np.float32)
    rc = load().dor_coverage_probe(C.c_uint32(len(splats)), _p(splats), C.byref(s), _p(xy), _p(sd), _p(zd), _p(out))
    assert rc == 0, rc
    return out
