"""Inputs of bgs_render_scene's tests (tests/test_oracle_scene.py, tests/test_gpu_scene.py): small seeded clouds placed
in front of the headless camera, transforms, splits into contiguous pieces, and each listed cloud as the scene oracle
reads it."""
from __future__ import annotations

import numpy as np

import bevy_gaussian_splatting_b200 as B


def cloud_in_box(n: int, seed: int, centre=(0.0, 1.5, -4.0), half=1.5, scale=0.06, sh_degree: int = 3) -> B.PlanarGaussian3d:
    """n gaussians in a cube of half-side `half` around `centre`, scales shrunk by `scale`; a few are deselected (w = 0)
    so that the draw modes have something to tell apart."""
    c = B.random_gaussians_3d_seeded(n, seed, sh_degree=sh_degree)
    pos = c.position_visibility.copy()
    pos[:, :3] = pos[:, :3] * np.float32(half / 20.0) + np.asarray(centre, np.float32)
    pos[::7, 3] = 0.0
    so = c.scale_opacity.copy()
    so[:, :3] *= np.float32(scale)
    return B.PlanarGaussian3d(pos, c.spherical_harmonic, c.rotation, so)


def transform(t=(0.0, 0.0, 0.0), s: float = 1.0, yaw: float = 0.0) -> B.CloudTransform:
    """A CloudTransform: rotation by `yaw` about +Y, uniform scale `s`, then translation `t`."""
    cy, sy = np.cos(yaw), np.sin(yaw)
    m = np.eye(4, dtype=np.float32)
    m[:3, :3] = np.array([[cy, 0.0, sy], [0.0, 1.0, 0.0], [-sy, 0.0, cy]], np.float32) * np.float32(s)
    m[:3, 3] = t
    return B.CloudTransform(m)


def split_points(n: int, k: int, seed: int = 0) -> list[int]:
    """k contiguous pieces of [0, n): the k - 1 interior cut points, uneven and never empty."""
    if k == 1:
        return []
    rng = np.random.default_rng(seed + 17 * k)
    return sorted(rng.choice(np.arange(1, n), size=k - 1, replace=False).tolist())


def pieces(n: int, k: int, seed: int = 0) -> list[np.ndarray]:
    cuts = [0] + split_points(n, k, seed) + [n]
    return [np.arange(a, b) for a, b in zip(cuts[:-1], cuts[1:])]


def oracle_cloud(cloud: B.PlanarGaussian3d, layout: str) -> B.PlanarGaussian3d:
    """The planes the oracle reads for `cloud` stored in `layout` ("f32", "f16" or "cov"), at SH degree 3."""
    c = cloud.with_sh_degree(3)
    if layout == "f16":
        return c.rounded_to_f16()
    if layout == "cov":
        return c.precomputed_covariance().rounded_to_f16()
    return c
