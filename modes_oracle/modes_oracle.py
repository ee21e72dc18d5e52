"""ctypes loader for the Classification / OpticalFlow colour oracle (modes_oracle/libmodes_oracle.so).  TEST
INFRASTRUCTURE ONLY.

May be imported only by tests/ and scripts/.  See modes_oracle.h for the rule.  `project_ex` composes a record of either
mode: oracle/'s Color-mode record (geometry, opacity, bbox, and the SH colour Classification starts from) with this
library's colour.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmodes_oracle.so")

CLASSIFICATION, OPTICAL_FLOW = 4, 5
HIGHLIGHT = np.array([0.3, 1.0, 0.1], np.float32)   # DrawMode::HighlightSelected (gaussian.wgsl:423-427)

_lib = None
_F = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")


def build() -> None:
    subprocess.run(["make", "-C", _HERE, "-s"], check=True)


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        lib = C.CDLL(LIB_PATH)
        lib.mo_hsv_to_rgb.argtypes = [C.c_uint32, _F, _F, _F, _F]
        lib.mo_atan2.argtypes = [C.c_uint32, _F, _F, _F]
        lib.mo_class_colour.argtypes = [C.c_uint32, _F, _F, C.c_uint32, _F]
        lib.mo_flow_colour.argtypes = [C.c_uint32, _F, _F, _F, _F, C.c_float, _F]
        for f in (lib.mo_hsv_to_rgb, lib.mo_atan2, lib.mo_class_colour, lib.mo_flow_colour):
            f.restype = None
        _lib = lib
    return _lib


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, np.float32)
    return a if shape is None else a.reshape(shape)


def hsv_to_rgb(h, s, v) -> np.ndarray:
    h, s, v = (_f32(np.broadcast_to(x, np.shape(h))).ravel() for x in (h, s, v))
    out = np.empty((len(h), 3), np.float32)
    load().mo_hsv_to_rgb(len(h), h, s, v, out)
    return out


def atan2(y, x) -> np.ndarray:
    y, x = _f32(y).ravel(), _f32(x).ravel()
    out = np.empty(len(y), np.float32)
    load().mo_atan2(len(y), y, x, out)
    return out


def class_colour(sh_rgb, vis, num_classes: int) -> np.ndarray:
    sh_rgb, vis = _f32(sh_rgb, (-1, 3)), _f32(vis).ravel()
    out = np.empty((len(vis), 3), np.float32)
    load().mo_class_colour(len(vis), sh_rgb, vis, num_classes, out)
    return out


def flow_colour(pos_vis, transform, clip_from_world, previous_clip_from_world, delta_time: float) -> np.ndarray:
    """`transform` / `clip_from_world` / `previous_clip_from_world`: 16 floats, column-major (the ABI's order)."""
    pos_vis = _f32(pos_vis, (-1, 4))
    out = np.empty((len(pos_vis), 3), np.float32)
    load().mo_flow_colour(len(pos_vis), pos_vis, _f32(transform).ravel(), _f32(clip_from_world).ravel(),
                          _f32(previous_clip_from_world).ravel(), float(delta_time), out)
    return out


def project_ex(oracle, cloud, view, uniform, settings, extras, ids) -> np.ndarray:
    """The records of `ids` in settings.rasterize_mode (Classification or OpticalFlow): oracle.project's Color-mode
    records with r, g, b replaced on every drawn record.  `extras`: an abi.bgs_render_extras."""
    mode = int(settings.rasterize_mode)
    s = type(settings).from_buffer_copy(bytes(settings))
    s.rasterize_mode = 0
    rec = oracle.project(cloud, view, uniform, s, ids)
    drawn = rec["xlo"] <= rec["xhi"]
    pv = cloud.position_visibility[np.asarray(ids, np.int64)]
    if mode == CLASSIFICATION:
        rgb = class_colour(np.stack([rec["r"], rec["g"], rec["b"]], 1), pv[:, 3], int(extras.num_classes))
    else:
        rgb = flow_colour(pv, np.asarray(uniform.transform), np.asarray(view.clip_from_world),
                          np.asarray(extras.previous_clip_from_world), extras.delta_time)
    lit = (int(settings.draw_mode) == 2) & (pv[:, 3] > 0.5)
    rgb[lit] = HIGHLIGHT
    for j, k in enumerate("rgb"):
        rec[k][drawn] = rgb[drawn, j]
    return rec
