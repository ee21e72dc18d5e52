"""Cameras and the Bevy `View` uniform fields the path reads.

`GaussianCamera` mirrors src/camera.rs:6-9.  The matrices are what Bevy 0.19 puts in its `View`
uniform for a `Camera3d` with the default `PerspectiveProjection` (fov pi/4, near 0.1, infinite
reverse-Z: glam's `perspective_infinite_reverse_rh`), all arithmetic in f32, column-major
(SURVEY.md §8c: this type lives in the bevy crate, not in the reference tree; the C ABI takes the
matrices as inputs so production parity does not depend on this harness).
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np

from . import abi


@dataclasses.dataclass
class GaussianCamera:  # src/camera.rs:6-9
    warmup: bool = False


def perspective_infinite_reverse_rh(fov_y: float, aspect: float, z_near: float) -> np.ndarray:
    f = np.float32(1.0) / np.float32(math.tan(0.5 * fov_y))
    m = np.zeros((4, 4), np.float32)  # m[row, col]
    m[0, 0] = f / np.float32(aspect)
    m[1, 1] = f
    m[3, 2] = -1.0
    m[2, 3] = z_near
    return m


def look_at_rh(eye, target, up) -> np.ndarray:
    """view_from_world for a camera at `eye` looking at `target` (Bevy: -Z forward, +Y up)."""
    eye = np.asarray(eye, np.float32); target = np.asarray(target, np.float32); up = np.asarray(up, np.float32)
    fwd = target - eye
    fwd = fwd / np.float32(np.linalg.norm(fwd))
    right = np.cross(fwd, up); right = right / np.float32(np.linalg.norm(right))
    true_up = np.cross(right, fwd)
    m = np.eye(4, dtype=np.float32)
    m[0, :3] = right; m[1, :3] = true_up; m[2, :3] = -fwd
    m[0, 3] = -np.dot(right, eye); m[1, 3] = -np.dot(true_up, eye); m[2, 3] = np.dot(fwd, eye)
    return m.astype(np.float32)


@dataclasses.dataclass
class View:
    """Row-major numpy matrices [row, col]; `to_abi` flattens them column-major as Bevy stores them."""

    view_from_world: np.ndarray
    clip_from_view: np.ndarray
    world_position: np.ndarray
    width: int
    height: int

    @property
    def clip_from_world(self) -> np.ndarray:
        return (self.clip_from_view.astype(np.float32) @ self.view_from_world.astype(np.float32)).astype(np.float32)

    def to_abi(self) -> abi.bgs_view:
        key = (self.view_from_world.tobytes(), self.clip_from_view.tobytes(), bytes(np.asarray(self.world_position, np.float32)),
               self.width, self.height)
        cached = getattr(self, "_abi_cache", None)
        if cached is not None and cached[0] == key:
            return cached[1]
        v = abi.bgs_view()
        v.view_from_world[:] = self.view_from_world.astype(np.float32).T.reshape(-1).tolist()
        v.clip_from_view[:] = self.clip_from_view.astype(np.float32).T.reshape(-1).tolist()
        v.clip_from_world[:] = self.clip_from_world.T.reshape(-1).tolist()
        v.world_position[:] = np.asarray(self.world_position, np.float32).tolist()
        v.viewport[:] = [0.0, 0.0, float(self.width), float(self.height)]
        self._abi_cache = (key, v)
        return v


def perspective_view(eye, target, width: int, height: int, fov_y: float = math.pi / 4, near: float = 0.1,
                     up=(0.0, 1.0, 0.0)) -> View:
    return View(look_at_rh(eye, target, up), perspective_infinite_reverse_rh(fov_y, width / height, near),
                np.asarray(eye, np.float32), int(width), int(height))


def headless_view(width: int = 1920, height: int = 1080) -> View:
    """examples/headless.rs:177-184: Camera3d at (0, 1.5, 5), identity rotation (looking -Z)."""
    return perspective_view((0.0, 1.5, 5.0), (0.0, 1.5, 4.0), width, height)


def orbit_view(index: int, count: int, width: int = 1920, height: int = 1080, radius: float = 5.0,
               centre=(0.0, 1.5, 0.0)) -> View:
    """Config C5 (SURVEY.md §8d): `count` cameras on a circle of radius 5 around (0, 1.5, 0)."""
    a = 2.0 * math.pi * index / max(count, 1)
    eye = (centre[0] + radius * math.sin(a), centre[1], centre[2] + radius * math.cos(a))
    return perspective_view(eye, centre, width, height)


def _quat_from_rotation(r: np.ndarray) -> np.ndarray:
    """(w, x, y, z), unit, of the rotation matrix r (3x3, float64)."""
    t = np.trace(r)
    if t > 0.0:
        s = 2.0 * math.sqrt(1.0 + t)
        return np.array([0.25 * s, (r[2, 1] - r[1, 2]) / s, (r[0, 2] - r[2, 0]) / s, (r[1, 0] - r[0, 1]) / s])
    i = int(np.argmax(np.diag(r)))
    j, k = (i + 1) % 3, (i + 2) % 3
    s = 2.0 * math.sqrt(1.0 + r[i, i] - r[j, j] - r[k, k])
    q = np.empty(4)
    q[0] = (r[k, j] - r[j, k]) / s
    q[1 + i] = 0.25 * s
    q[1 + j] = (r[j, i] + r[i, j]) / s
    q[1 + k] = (r[k, i] + r[i, k]) / s
    return q / np.linalg.norm(q)


def _rotation_from_quat(q: np.ndarray) -> np.ndarray:
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def interpolate_view(a: View, b: View, u: float) -> View:
    """The camera a fraction `u` of the way from `a` to `b`, for the sub-frames of a shutter (`render_shutter`): the eye
    is lerped, a + u (b - a); the orientation is the shortest-arc slerp, from a's to b's, of the rotations of the two
    view_from_world matrices; the projection, width and height are a's.  Computed in float64 and stored in f32.  u = 0
    gives a's eye and view_from_world exactly, u = 1 b's."""
    u = float(u)
    ea, eb = np.asarray(a.world_position, np.float64), np.asarray(b.world_position, np.float64)
    eye = ((1.0 - u) * ea + u * eb).astype(np.float32)
    if u == 0.0 or u == 1.0:
        return View((a if u == 0.0 else b).view_from_world.copy(), a.clip_from_view.copy(), eye, a.width, a.height)
    qa = _quat_from_rotation(a.view_from_world[:3, :3].astype(np.float64))
    qb = _quat_from_rotation(b.view_from_world[:3, :3].astype(np.float64))
    d = float(np.dot(qa, qb))
    if d < 0.0:   # (the shorter arc)
        qb, d = -qb, -d
    if d > 1.0 - 1e-12:
        q = qa + u * (qb - qa)
    else:
        th = math.acos(d)
        q = (math.sin((1.0 - u) * th) * qa + math.sin(u * th) * qb) / math.sin(th)
    r = _rotation_from_quat(q / np.linalg.norm(q))
    m = np.eye(4, dtype=np.float32)
    m[:3, :3] = r
    m[:3, 3] = -(r @ eye.astype(np.float64))
    return View(m, a.clip_from_view.copy(), eye, a.width, a.height)


def shutter_times(time: float, shutter: float, count: int) -> np.ndarray:
    """The `count` sample times of a shutter of length `shutter` centred on `time`: the midpoints of its `count` equal
    parts, time + shutter ((i + 0.5) / count - 0.5) for i = 0 .. count - 1, each operation in f32.  For the uniforms'
    `time` of a `render_shutter` call's samples."""
    if count < 1:
        raise ValueError(f"shutter_times: count = {count}, at least 1")
    i = np.arange(count, dtype=np.float32)
    f32 = np.float32
    return (f32(time) + f32(shutter) * ((i + f32(0.5)) / f32(count) - f32(0.5))).astype(np.float32)
