"""ctypes loader for the CPU oracle (oracle/liboracle.so).  TEST INFRASTRUCTURE ONLY.

May be imported only by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs.  See oracle/bgs_oracle.h for the parity status and FP policy.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liboracle.so")


class orc_view(C.Structure):
    _fields_ = [("view_from_world", C.c_float * 16), ("clip_from_view", C.c_float * 16),
                ("clip_from_world", C.c_float * 16), ("world_position", C.c_float * 3), ("viewport", C.c_float * 4)]


class orc_uniform(C.Structure):
    _fields_ = [("transform", C.c_float * 16), ("global_opacity", C.c_float), ("global_scale", C.c_float),
                ("color_space", C.c_uint32), ("time", C.c_float), ("aabb_min", C.c_float * 4), ("aabb_max", C.c_float * 4)]


class orc_settings(C.Structure):
    _fields_ = [("gaussian_mode", C.c_uint32), ("rasterize_mode", C.c_uint32), ("aabb", C.c_uint32),
                ("opacity_adaptive_radius", C.c_uint32), ("draw_mode", C.c_uint32),
                ("radix_sort_depth_bits", C.c_uint32), ("flags", C.c_uint32), ("reserved", C.c_uint32)]


SPLAT_DTYPE = np.dtype([("cx", "f4"), ("cy", "f4"), ("ux", "f4"), ("uy", "f4"), ("vx", "f4"), ("vy", "f4"),
                        ("r", "f4"), ("g", "f4"), ("b", "f4"), ("op", "f4"),
                        ("xlo", "i4"), ("xhi", "i4"), ("ylo", "i4"), ("yhi", "i4"), ("extra", "f4", (16,))])
assert SPLAT_DTYPE.itemsize == 120

_lib = None


def build() -> None:
    subprocess.run(["make", "-C", _HERE, "-s"], check=True)


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        _lib = C.CDLL(LIB_PATH)
        _lib.orc_cpu_sort_model.restype = C.c_double
        _lib.orc_ln.restype = C.c_float
        _lib.orc_ln.argtypes = [C.c_float]
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _conv(src, cls):
    """Reinterpret a same-layout ctypes struct (e.g. bgs_view) as the oracle's struct."""
    if isinstance(src, cls):
        return src
    assert C.sizeof(src) == C.sizeof(cls)
    return cls.from_buffer_copy(bytes(src))


def pass_plan(depth_bits: int):
    a, b, c = C.c_uint32(), C.c_uint32(), C.c_uint32()
    load().orc_pass_plan(C.c_uint32(depth_bits), C.byref(a), C.byref(b), C.byref(c))
    return a.value, b.value, c.value


def keygen(pos_vis: np.ndarray, view, uniform, depth_bits: int = 32) -> np.ndarray:
    n = len(pos_vis)
    out = np.empty(n, np.uint32)
    v, u = _conv(view, orc_view), _conv(uniform, orc_uniform)
    rc = load().orc_keygen(C.c_uint32(n), _p(pos_vis), C.byref(v), C.byref(u), C.c_uint32(depth_bits), _p(out))
    assert rc == 0
    return out


def radix_sort(keys: np.ndarray, depth_bits: int = 32):
    n = len(keys)
    sk, si = np.empty(n, np.uint32), np.empty(n, np.uint32)
    rc = load().orc_radix_sort(C.c_uint32(n), _p(np.ascontiguousarray(keys, np.uint32)), C.c_uint32(depth_bits), _p(sk), _p(si))
    assert rc == 0, rc
    return sk, si


def stable_sort(keys: np.ndarray) -> np.ndarray:
    n = len(keys)
    si = np.empty(n, np.uint32)
    load().orc_stable_sort(C.c_uint32(n), _p(np.ascontiguousarray(keys, np.uint32)), _p(si))
    return si


def pack_f16(sh, rot, so):
    n = len(sh)
    shp, rso = np.empty((n, 24), np.uint32), np.empty((n, 4), np.uint32)
    load().orc_pack_f16(C.c_uint32(n), _p(sh), _p(rot), _p(so), _p(shp), _p(rso))
    return shp, rso


def decode_f16(shp, rso):
    n = len(shp)
    sh, rot, so = np.empty((n, 48), np.float32), np.empty((n, 4), np.float32), np.empty((n, 4), np.float32)
    load().orc_decode_f16(C.c_uint32(n), _p(shp), _p(rso), _p(sh), _p(rot), _p(so))
    return sh, rot, so


def covariance_3d(rot: np.ndarray, so: np.ndarray) -> np.ndarray:
    n = len(rot)
    out = np.empty((n, 6), np.float32)
    load().orc_covariance_3d(C.c_uint32(n), _p(np.ascontiguousarray(rot, np.float32)), _p(np.ascontiguousarray(so, np.float32)), _p(out))
    return out


def project(cloud, view, uniform, settings, ids: np.ndarray) -> np.ndarray:
    ids = np.ascontiguousarray(ids, np.uint32)
    out = np.zeros(len(ids), SPLAT_DTYPE)
    v, u, s = _conv(view, orc_view), _conv(uniform, orc_uniform), _conv(settings, orc_settings)
    rc = load().orc_project(C.c_uint32(len(cloud)), _p(cloud.position_visibility), _p(cloud.spherical_harmonic),
                            _p(cloud.rotation), _p(cloud.scale_opacity), C.byref(v), C.byref(u), C.byref(s),
                            C.c_uint32(len(ids)), _p(ids), _p(out))
    assert rc == 0
    return out


def render_ref(cloud, view, uniform, settings, threads: int = 0, dst: np.ndarray | None = None) -> np.ndarray:
    """ref_mode frame.  `dst`: (H, W, 4) f32 premultiplied target to blend over (None = opaque black clear)."""
    v, u, s = _conv(view, orc_view), _conv(uniform, orc_uniform), _conv(settings, orc_settings)
    W, H = int(v.viewport[2]), int(v.viewport[3])
    out = np.empty((H, W, 4), np.float32)
    if dst is not None:
        dst = np.ascontiguousarray(dst, np.float32)
        assert dst.shape == (H, W, 4)
    rc = load().orc_render_ref_over(C.c_uint32(len(cloud)), _p(cloud.position_visibility), _p(cloud.spherical_harmonic),
                                    _p(cloud.rotation), _p(cloud.scale_opacity), C.byref(v), C.byref(u), C.byref(s), _p(dst), _p(out),
                                    C.c_int(threads))
    assert rc == 0
    return out


def render_tiles(cloud, view, uniform, settings, want_image: bool = True, threads: int = 0):
    """-> dict(image, tile_ranges (T,2), tile_entries (I,), n_pairs, n_vis, rank_to_id)."""
    v, u, s = _conv(view, orc_view), _conv(uniform, orc_uniform), _conv(settings, orc_settings)
    W, H = int(v.viewport[2]), int(v.viewport[3])
    T = ((W + 15) // 16) * ((H + 15) // 16)
    n = len(cloud)
    args = (C.c_uint32(n), _p(cloud.position_visibility), _p(cloud.spherical_harmonic), _p(cloud.rotation),
            _p(cloud.scale_opacity), C.byref(v), C.byref(u), C.byref(s))
    n_pairs, n_vis = C.c_uint64(), C.c_uint32()
    ranges = np.empty((T, 2), np.uint32)
    # first call: counts only
    rc = load().orc_render_tiles(*args, None, _p(ranges), None, C.c_uint64(0), C.byref(n_pairs), C.byref(n_vis), None,
                                 C.c_int(threads))
    assert rc == 0
    entries = np.empty(n_pairs.value, np.uint32)
    r2i = np.empty(n_vis.value, np.uint32)
    img = np.empty((H, W, 4), np.float32) if want_image else None
    rc = load().orc_render_tiles(*args, _p(img), _p(ranges), _p(entries), C.c_uint64(n_pairs.value), C.byref(n_pairs),
                                 C.byref(n_vis), _p(r2i), C.c_int(threads))
    assert rc == 0
    return dict(image=img, tile_ranges=ranges, tile_entries=entries, n_pairs=n_pairs.value, n_vis=n_vis.value,
                rank_to_id=r2i)


PROBE_DTYPE = np.dtype([("u", "f4"), ("v", "f4"), ("mx", "f4"), ("my", "f4"), ("Rq", "f4"), ("power", "f4"), ("alpha", "f4"),
                        ("covered", "u4"), ("covered_if_unfused", "u4")])
TRACE_DTYPE = np.dtype([("c64", "f8", (3,)), ("T64", "f8"), ("t_sens", "f8"), ("stop_margin", "f8"), ("w_power", "f8"),
                        ("t_sens_power", "f8"), ("T", "f4"),
                        ("n_blended", "u4"), ("rank0", "i4"), ("rank1", "i4"), ("flags", "u4"), ("max_c", "f4"),
                        ("max_power", "f4"), ("pad", "u4")])
assert TRACE_DTYPE.itemsize == 96
TRACE_NEAR_STOP, TRACE_NEAR_CLAMP, TRACE_UNCLAMPED = 1, 2, 4


def coverage_probe(splats: np.ndarray, settings, pixel_xy: np.ndarray) -> np.ndarray:
    """`splats`: SPLAT_DTYPE records; `pixel_xy`: (len(splats), 2) pixel centres -> PROBE_DTYPE per pair."""
    splats = np.ascontiguousarray(splats, SPLAT_DTYPE)
    xy = np.ascontiguousarray(pixel_xy, np.float32).reshape(len(splats), 2)
    out = np.zeros(len(splats), PROBE_DTYPE)
    s = _conv(settings, orc_settings)
    rc = load().orc_coverage_probe(C.c_uint32(len(splats)), _p(splats), C.byref(s), _p(xy), _p(out))
    assert rc == 0
    return out


def blend_trace(cloud, view, uniform, settings, threads: int = 0) -> np.ndarray:
    """-> (H, W) TRACE_DTYPE: render_tiles' walk per pixel, with its blend also evaluated in float64."""
    v, u, s = _conv(view, orc_view), _conv(uniform, orc_uniform), _conv(settings, orc_settings)
    W, H = int(v.viewport[2]), int(v.viewport[3])
    out = np.zeros((H, W), TRACE_DTYPE)
    rc = load().orc_blend_trace(C.c_uint32(len(cloud)), _p(cloud.position_visibility), _p(cloud.spherical_harmonic),
                                _p(cloud.rotation), _p(cloud.scale_opacity), C.byref(v), C.byref(u), C.byref(s), _p(out),
                                C.c_int(threads))
    assert rc == 0
    return out


def cpu_sort_model(pos_vis: np.ndarray, cam, threads: int = 0) -> float:
    cam = np.asarray(cam, np.float32)
    return float(load().orc_cpu_sort_model(C.c_uint32(len(pos_vis)), _p(pos_vis), _p(cam), C.c_int(threads), None))


def num_threads() -> int:
    return int(load().orc_num_threads())
