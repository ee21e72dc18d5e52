"""Cases for bgs_cloud_transform and bgs_cloud_bounds (include/bgs.h): the matrices the call accepts and refuses, and
clouds whose gaussians reach every class of the rule -- unit and non-unit quaternions; zero, subnormal and huge scales;
positions that are -0, +-inf or NaN; visibility at 0.5, just below it, NaN, +-inf and -0 -- in every layout (f32, f16,
f16 precomputed covariance) and SH degree 0..3."""
from __future__ import annotations

import numpy as np

import bevy_gaussian_splatting_b200 as B

F = np.float32
LAYOUTS = ("f32", "f16", "cov")
DEGREES = (0, 1, 2, 3)


def _rot(axis, angle):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    h = 0.5 * angle
    return (np.cos(h), *(np.sin(h) * a))


def _exact_turn(axis: int) -> np.ndarray:
    """An exact 90-degree turn about one axis: every entry 0 or +-1."""
    m = np.eye(4, dtype=F)
    i, j = [(1, 2), (2, 0), (0, 1)][axis]
    m[i, i] = m[j, j] = 0.0
    m[i, j], m[j, i] = -1.0, 1.0
    return m


def _general() -> np.ndarray:
    return B.similarity_transform((1.5, -2.25, 0.75), _rot((0.3, -0.8, 0.5), 1.1), 1.7, (0.5, 0.25, -1.0))


def _scaled_column(eps: float) -> np.ndarray:
    """The general matrix with its first column scaled by (1 + eps): |c0|^2 - s^2 is about (4/3) eps s^2."""
    m = _general().astype(np.float64)
    m[:3, 0] *= 1.0 + eps
    return m.astype(F)


# the matrices the call accepts (4x4, CloudTransform.matrix's convention)
ACCEPTED = {
    "identity": np.eye(4, dtype=F),
    "translation": B.similarity_transform((3.0, -1.5, 0.25)),
    "turn_x": _exact_turn(0),
    "turn_y": _exact_turn(1),
    "turn_z": _exact_turn(2),
    "general": _general(),
    "tolerance_inside": _scaled_column(7.0e-6),
}


def _refused():
    out = {}
    m = np.eye(4, dtype=F); m[0, 1] = 0.2
    out["shear"] = m
    out["non_uniform"] = np.diag([1.0, 2.0, 1.0, 1.0]).astype(F)
    out["reflection"] = np.diag([-1.0, 1.0, 1.0, 1.0]).astype(F)
    out["reflection_general"] = (_general() @ np.diag([1.0, 1.0, -1.0, 1.0]).astype(F)).astype(F)
    m = np.eye(4, dtype=F); m[3, 0] = 0.5
    out["non_affine"] = m
    m = np.eye(4, dtype=F); m[3, 3] = 2.0
    out["bottom_row_w"] = m
    m = _general().copy(); m[1, 2] = np.nan
    out["nan_entry"] = m
    m = _general().copy(); m[0, 3] = np.inf
    out["inf_entry"] = m
    out["zero"] = np.diag([0.0, 0.0, 0.0, 1.0]).astype(F)
    out["tolerance_outside"] = _scaled_column(1.2e-5)
    return out


REFUSED = _refused()

# visibility values whose selection the predicate !(v < 0.5) decides
SPECIAL_VIS = np.array([0.5, np.nextafter(F(0.5), F(0)), np.nan, np.inf, -np.inf, -0.0, 1.0, 0.0], F)


def cloud(n: int, degree: int, seed: int, unit: bool = True, special: bool = True) -> B.PlanarGaussian3d:
    """A cloud of n gaussians at the SH degree: random positions, half of them selected, unit quaternions (or the raw
    non-unit draws), and, with `special`, the first rows set to the classes the rule names."""
    c = B.random_gaussians_3d_seeded(n, seed, sh_degree=degree)
    rng = np.random.default_rng(seed)
    c.position_visibility[:, 3] = (rng.random(n) < 0.5).astype(F)
    if unit:
        c.rotation /= np.linalg.norm(c.rotation, axis=1, keepdims=True)
    if special:
        p, so = c.position_visibility, c.scale_opacity
        k = len(SPECIAL_VIS)
        p[:k, 3] = SPECIAL_VIS
        p[k + 0, :3] = (-0.0, -0.0, -0.0)
        p[k + 1, 0] = np.inf
        p[k + 2, 1] = -np.inf
        p[k + 3, 2] = np.nan
        p[k + 4, :3] = (np.nan, np.inf, -np.inf)
        so[k + 5, :3] = 0.0
        so[k + 6, :3] = (1e-40, 3e-45, 1e-39)     # subnormal
        so[k + 7, :3] = (3e38, 1e30, 6e4)         # huge (f16: past 65504 after the scale)
        c.rotation[k + 8] = (0.0, 0.0, 0.0, 0.0)
        c.rotation[k + 9] = (2.0, -1.0, 0.5, 3.0)  # non-unit
        p[k:k + 10, 3] = 1.0
    return c


def planes_of(c: B.PlanarGaussian3d, layout: str):
    """The upload planes of the layout: f32 (pos_vis, sh, rot, scale_opacity); f16 and cov (pos_vis, sh_packed,
    second plane)."""
    if layout == "f32":
        return (c.position_visibility, c.spherical_harmonic, c.rotation, c.scale_opacity)
    src = c.precomputed_covariance() if layout == "cov" else c
    sh, second = src.pack_f16()
    return (c.position_visibility, sh, second)


def selected(vis) -> np.ndarray:
    """The transform's and the bounds' predicate: !(v < 0.5)."""
    return ~(np.asarray(vis, F) < F(0.5))


def bounds(pos_vis, selected_only: bool):
    """bgs_cloud_bounds restated in numpy: (min, max, count) over the gaussians with finite x, y, z (and selected)."""
    p = np.asarray(pos_vis, F)
    keep = np.all(np.isfinite(p[:, :3]), axis=1)
    if selected_only:
        keep &= selected(p[:, 3])
    if not keep.any():
        return np.full(3, np.inf, F), np.full(3, -np.inf, F), 0
    q = p[keep, :3]
    return q.min(0), q.max(0), int(keep.sum())


def mat4_point(M, pos_vis) -> np.ndarray:
    """(n, 3) f32: the projection's model multiply of the positions, ((m_r0 x + m_r1 y) + m_r2 z) + m_r3 per row."""
    M, p = np.asarray(M, F), np.asarray(pos_vis, F)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    with np.errstate(all="ignore"):
        return np.stack([((M[r, 0] * x + M[r, 1] * y) + M[r, 2] * z) + M[r, 3] for r in range(3)], 1).astype(F)
