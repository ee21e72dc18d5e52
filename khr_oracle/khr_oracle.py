"""CPU restatement of the reference's KHR_gaussian_splatting attribute readers (src/io/scene.rs:1305-2015:
read_*_attribute, normalize_*, normalize_quaternion, the SH map's placement and the COLOR_0 fallback) over the accessor
descriptors `B.load_scene` produces.  Test infrastructure only: the product never imports it.

Every f32 operation is numpy float32 in the reference's order (numpy neither fuses nor reorders elementwise ops); exp is
evaluated in f64 and rounded once to f32, as bgs_cloud_upload_khr does (f32 expf is only good to 2 ulp).
"""
from __future__ import annotations

import numpy as np

from bevy_gaussian_splatting_b200.gaussian import SH_WIDTHS, PlanarGaussian3d

F = np.float32
SH_DEGREE_ZERO_BASIS = F(0.282095)
# accepted (components, component type, normalised) per slot: normalised None = either
ACCEPTED = {
    "POSITION": (3, {5126: None}),
    "ROTATION": (4, {5126: None, 5120: True, 5122: True}),
    "SCALE": (3, {5126: None, 5120: None, 5122: None}),
    "OPACITY": (1, {5126: None, 5121: True, 5123: True}),
    "COLOR_0": ((3, 4), {5126: None, 5121: None, 5123: None}),
    "SH": (3, {5126: None}),
}


def _check(slot: str, a) -> None:
    comps, types = ACCEPTED[slot]
    ok = a.components in (comps if isinstance(comps, tuple) else (comps,)) and a.component_type in types
    if ok and types[a.component_type] is not None and bool(a.normalized) != types[a.component_type]:
        ok = False
    if not ok:
        raise ValueError(f"{slot} does not accept {a.components} components of component type {a.component_type} "
                         f"(normalized {a.normalized})")


def read(a) -> np.ndarray:
    """The accessor's values as f32 (count, components): normalize_i8 / _i16 / _u8 / _u16 where the reference applies them
    (u8 / u16 always read as normalised; they are accepted only where that is the reference's reading)."""
    v = a.array()
    t = a.component_type
    if t == 5126:
        return v.astype(F)
    x = v.astype(F)
    if t == 5120:
        return np.maximum(x / F(127.0), F(-1.0)) if a.normalized else x
    if t == 5122:
        return np.maximum(x / F(32767.0), F(-1.0)) if a.normalized else x
    return x / (F(255.0) if t == 5121 else F(65535.0))


def normalize_quaternions(q: np.ndarray) -> tuple[np.ndarray, int]:
    """normalize_quaternion (scene.rs:1979-1999) per row: ((q0 q0 + q1 q1) + q2 q2) + q3 q3, then sqrt, 1 / x, multiply;
    a length^2 <= FLT_EPSILON becomes (1, 0, 0, 0).  Returns (quaternions, how many were replaced)."""
    q = np.asarray(q, F)
    l2 = ((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2]) + q[:, 3] * q[:, 3]
    zero = l2 <= np.finfo(F).eps
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        inv = F(1.0) / np.sqrt(l2)
        out = (q * inv[:, None]).astype(F)
    out[zero] = np.array([1, 0, 0, 0], F)
    return out, int(zero.sum())


def exp_f32(raw: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore"):
        return np.exp(np.asarray(raw, F).astype(np.float64)).astype(F)


def decode(prim) -> tuple[PlanarGaussian3d, int]:
    """(the decoded cloud at the primitive's SH degree, zero-length quaternions replaced); ValueError for each value or
    accessor the reference refuses."""
    for slot, a in (("POSITION", prim.position), ("ROTATION", prim.rotation), ("SCALE", prim.scale), ("OPACITY", prim.opacity)):
        _check(slot, a)
    for a in prim.sh:
        _check("SH", a)
    use_color = not prim.sh and prim.color_0 is not None
    if use_color:
        _check("COLOR_0", prim.color_0)
    n = prim.n
    pos = read(prim.position)
    if not np.isfinite(pos).all():
        raise ValueError("POSITION contains non-finite values")
    rot, zero = normalize_quaternions(read(prim.rotation))
    if not np.isfinite(rot).all():
        raise ValueError("ROTATION is non-finite after normalising")
    scale = exp_f32(read(prim.scale))
    if not np.isfinite(scale).all():
        raise ValueError("SCALE gives a non-finite exp(scale)")
    op = read(prim.opacity)[:, 0]
    if not ((op >= 0) & (op <= 1)).all():
        raise ValueError("OPACITY is NaN or outside [0, 1]")
    degree = prim.sh_degree if prim.sh else 0
    sh = np.zeros((n, SH_WIDTHS[degree]), F)
    for k, a in enumerate(prim.sh):
        sh[:, 3 * k:3 * k + 3] = read(a)
    if not np.isfinite(sh).all():
        raise ValueError("an SH coefficient is non-finite")
    if use_color:
        color = read(prim.color_0)[:, :3]
        if not np.isfinite(color).all():
            raise ValueError("COLOR_0 contains non-finite values")
        sh[:, :3] = color / SH_DEGREE_ZERO_BASIS
    pv = np.empty((n, 4), F)
    pv[:, :3], pv[:, 3] = pos, F(1.0)
    so = np.empty((n, 4), F)
    so[:, :3], so[:, 3] = scale, op
    return PlanarGaussian3d(pv, sh, rot, so), zero
