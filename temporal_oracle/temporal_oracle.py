"""ctypes loader for the Gaussian4d frame oracle (temporal_oracle/libtemporal_oracle.so).  TEST INFRASTRUCTURE ONLY.

May be imported only by tests/ and scripts/.  See temporal_oracle.h for the rule.  `cloud`: a PlanarGaussian4d;
`view` / `uniform` / `settings` / `extras`: the ABI structs (abi.bgs_view, ...), converted like oracle/'s.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtemporal_oracle.so")

_lib = None


class tor_temporal(C.Structure):
    _fields_ = [("time_start", C.c_float), ("time_stop", C.c_float), ("prev_clip_from_world", C.c_float * 16),
                ("delta_time", C.c_float), ("num_classes", C.c_uint32)]


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


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, np.float32)
    return a if shape is None else a.reshape(shape)


def exp(x) -> np.ndarray:
    x = _f32(x).ravel()
    out = np.empty_like(x)
    load().tor_exp(C.c_uint32(len(x)), _p(x), _p(out))
    return out


def cos(x) -> np.ndarray:
    x = _f32(x).ravel()
    out = np.empty_like(x)
    load().tor_cos(C.c_uint32(len(x)), _p(x), _p(out))
    return out


def condition(rot8, so, tt, global_scale: float, t: float) -> dict:
    rot8, so, tt = _f32(rot8, (-1, 8)), _f32(so, (-1, 4)), _f32(tt, (-1, 4))
    n = len(rot8)
    cov6, dm, marg, mask = np.empty((n, 6), np.float32), np.empty((n, 3), np.float32), np.empty(n, np.float32), np.empty(n, np.uint8)
    load().tor_condition(C.c_uint32(n), _p(rot8), _p(so), _p(tt), C.c_float(global_scale), C.c_float(t), _p(cov6), _p(dm),
                         _p(marg), _p(mask))
    return dict(cov6=cov6, delta_mean=dm, marginal=marg, mask=mask.astype(bool))


def temporal(time_start: float, time_stop: float, extras=None) -> tor_temporal:
    tp = tor_temporal(time_start=time_start, time_stop=time_stop, num_classes=1)
    if extras is not None:
        tp.prev_clip_from_world[:] = extras.previous_clip_from_world[:]
        tp.delta_time = extras.delta_time
        tp.num_classes = extras.num_classes
    return tp


def frame(cloud, view, uniform, settings, time_start: float, time_stop: float, extras=None, scene=None,
          want_image: bool = True, threads: int = 0) -> dict:
    """-> dict(records (n_vis, 12) in bgs_debug_projected's layout by rank, rank_to_id, depths, image (H, W, 4) or None)."""
    v, u, s = O._conv(view, O.orc_view), O._conv(uniform, O.orc_uniform), O._conv(settings, O.orc_settings)
    W, H = int(v.viewport[2]), int(v.viewport[3])
    tp = temporal(time_start, time_stop, extras)
    planes = [np.ascontiguousarray(a, np.float32) for a in cloud.planes()]
    pitch = 0
    if scene is not None:
        scene = np.ascontiguousarray(scene, np.float32)
        pitch = scene.shape[1] * 4
    nv = C.c_uint32()
    args = [C.c_uint32(len(cloud))] + [_p(a) for a in planes] + [C.byref(v), C.byref(u), C.byref(s), C.byref(tp), _p(scene),
                                                                 C.c_uint64(pitch), C.byref(nv)]
    assert load().tor_frame(*args, None, None, None, None, C.c_int(threads)) == 0
    n = nv.value
    rec, r2i, d = np.empty((n, 12), np.float32), np.empty(n, np.uint32), np.empty(n, np.float32)
    img = np.empty((H, W, 4), np.float32) if want_image else None
    assert load().tor_frame(*args, _p(rec), _p(r2i), _p(d), _p(img), C.c_int(threads)) == 0
    return dict(records=rec, rank_to_id=r2i, depths=d, image=img)
