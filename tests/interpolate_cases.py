"""Seeded interpolation cases for bgs_cloud_interpolate's tests (tests/test_oracle_interpolate.py on the CPU,
tests/test_gpu_interpolate.py on the H100): one case per class of input the rule in include/bgs.h distinguishes.

Each case is a dict: name, cls (its class), time, time_start, time_stop, same (rhs is lhs), and lhs / rhs: for each
layout ("f32", "f16", "cov") the planes its upload call takes (f32: pos_vis, sh, rot, scale_opacity; f16 and cov:
pos_vis, sh_packed, second plane).  Gaussian 0 of every case is the factor probe: every lhs lane 0, every rhs lane 1,
so its position lanes come out as t (+0 for t = -0).  Then come the class's special gaussians, then `fill` random
ones (`cases(fill)`: the GPU file reaches 200 000 gaussians with the same builders).
"""
from __future__ import annotations

import numpy as np

from bevy_gaussian_splatting_b200.gaussian import PlanarGaussian3d, random_gaussians_3d_seeded

F = np.float32
FMAX = float(np.finfo(F).max)
EPS_D = F(1e-6)                                        # interpolate.wgsl:53: `abs(duration) < 1e-6`
LAYOUTS = ("f32", "f16", "cov")

CLASSES = ("t_zero", "t_one", "t_clamped", "t_interior", "d_at_eps", "d_below_eps", "d_above_eps", "d_negative",
           "t_negative_zero", "time_eq_stop", "time_below_stop", "t_subnormal", "lanes", "lanes_t_zero", "same",
           "quaternions", "f16_halves")

# f32 lane values whose pairs the lane classes blend
LANE_VALUES = np.array([0.0, -0.0, 1e-45, 3e-45, -1.1e-38, 1.0, -2.5, 3.3e-3, FMAX, -FMAX, np.inf, -np.inf, np.nan], F)
# half bit patterns whose pairs the f16 class blends: zeros, subnormals, the largest finite, infinities, NaNs, and
# neighbours of 1 whose midpoints are round-to-nearest-even ties
HALF_VALUES = np.array([0x0000, 0x8000, 0x0001, 0x0002, 0x0003, 0x03FF, 0x8001, 0x7BFF, 0xFBFF, 0x7C00, 0xFC00, 0x7E00,
                        0x7C01, 0xFE00, 0x3C00, 0x3C01, 0x3C02, 0x3555], np.uint32)


def _f32_planes(c: PlanarGaussian3d):
    return (c.position_visibility, c.spherical_harmonic, c.rotation, c.scale_opacity)


def _layouts(c: PlanarGaussian3d):
    """The upload planes of one host cloud in every layout (f16 and cov: the same packed words, read as rotation-scale
    or as covariance records)."""
    with np.errstate(over="ignore", invalid="ignore"):
        sh, second = c.pack_f16()
    return {"f32": tuple(np.ascontiguousarray(a, F) for a in _f32_planes(c)),
            "f16": (np.ascontiguousarray(c.position_visibility, F), sh, second),
            "cov": (np.ascontiguousarray(c.position_visibility, F), sh.copy(), second.copy())}


def _cloud(n):
    return PlanarGaussian3d(np.zeros((n, 4), F), np.zeros((n, 48), F), np.zeros((n, 4), F), np.zeros((n, 4), F))


def _concat(*clouds):
    return PlanarGaussian3d(*(np.concatenate([_f32_planes(c)[k] for c in clouds]) for k in range(4)))


def _probe():
    lhs, rhs = _cloud(1), _cloud(1)
    for a in _f32_planes(rhs):
        a[:] = 1.0
    return lhs, rhs


def _fill(n, seed):
    return random_gaussians_3d_seeded(n, seed), random_gaussians_3d_seeded(n, seed + 1000)


def _pairs(values, count, seed):
    """count (lhs, rhs) pairs of `values`, every ordered pair at least once when count allows, then random ones."""
    k = len(values)
    a, b = np.meshgrid(np.arange(k), np.arange(k), indexing="ij")
    ia, ib = a.reshape(-1), b.reshape(-1)
    rng = np.random.default_rng(seed)
    reps = -(-count // len(ia))
    ia, ib = np.tile(ia, reps)[:count], np.tile(ib, reps)[:count]
    p = rng.permutation(count)
    return values[ia[p]], values[ib[p]]


def _lane_specials(seed, m=64):
    """m gaussians whose position, SH and scale-opacity lanes are every pair of LANE_VALUES; rotations plain."""
    lhs, rhs = _fill(m, seed)
    for k in (0, 1, 3):
        width = _f32_planes(lhs)[k].shape[1]
        a, b = _pairs(LANE_VALUES, m * width, seed + k)
        _f32_planes(lhs)[k][:] = a.reshape(m, width)
        _f32_planes(rhs)[k][:] = b.reshape(m, width)
    return lhs, rhs


def _quaternion_specials(seed):
    """Rotations for l2 == 0 (zero, -0, underflowing squares), l2 == inf (overflowing squares), NaN, inf, antipodal
    pairs (q and -q: zero at t = 0.5) and plain ones."""
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(8, 4)).astype(F)
    q /= np.linalg.norm(q, axis=1, keepdims=True).astype(F)
    rows_l = [[0, 0, 0, 0], [-0.0, -0.0, -0.0, -0.0], [1e-25, -1e-25, 1e-25, 1e-30], [1e20, 1e20, -1e20, 3e19],
              [np.nan, 0.5, 0.5, 0.5], [np.inf, 0, 0, 0], [0.5, -0.5, 0.5, -0.5], [-1e-3, 2e-3, 0, 0]]
    rows_r = [[0, 0, 0, 0], [-0.0, 0.0, -0.0, -0.0], [-1e-25, 1e-25, 1e-30, 1e-25], [1e20, -1e20, 1e20, 1e20],
              [0.5, 0.5, 0.5, 0.5], [1, 0, 0, 0], [-0.5, 0.5, -0.5, 0.5], [1e-3, -2e-3, 0, 0]]
    lhs, rhs = _fill(len(rows_l) + 16, seed)
    lhs.rotation[: len(rows_l)] = np.array(rows_l, F)
    rhs.rotation[: len(rows_r)] = np.array(rows_r, F)
    lhs.rotation[len(rows_l):len(rows_l) + 8] = q                  # antipodal pairs of unit quaternions
    rhs.rotation[len(rows_l):len(rows_l) + 8] = -q
    return lhs, rhs


def _half_specials(layouts_l, layouts_r, seed, m=64):
    """Overwrite m gaussians (from index 1) of the f16 and cov planes with every pair of HALF_VALUES, in every half of
    the SH words and of the second plane."""
    for lay in ("f16", "cov"):
        for plane in (1, 2):
            wl, wr = layouts_l[lay][plane], layouts_r[lay][plane]
            width = wl.shape[1]
            a, b = _pairs(HALF_VALUES, 2 * m * width, seed + plane)
            a, b = a.reshape(m, width, 2), b.reshape(m, width, 2)
            wl[1:1 + m] = (a[..., 0] << 16) | a[..., 1]
            wr[1:1 + m] = (b[..., 0] << 16) | b[..., 1]


def _case(name, cls, time, time_start, time_stop, lhs, rhs, same=False, halves=False, seed=0):
    L, R = _layouts(lhs), _layouts(rhs)
    if halves:
        _half_specials(L, R, seed)
    if same:
        R = L
    return {"name": name, "cls": cls, "time": float(F(time)), "time_start": float(F(time_start)),
            "time_stop": float(F(time_stop)), "same": same, "lhs": L, "rhs": R}


def cases(fill: int = 256):
    probe_l, probe_r = _probe()
    fl, fr = _fill(fill, 7)
    sl, sr = _lane_specials(11)
    base_l, base_r = _concat(probe_l, sl, fl), _concat(probe_r, sr, fr)
    below, above = np.nextafter(EPS_D, F(0)), np.nextafter(EPS_D, F(1))
    out = []
    factor = [("t_zero", 0.0, 0.0, 1.0), ("t_one", 1.0, 0.0, 1.0), ("t_clamped", -0.5, 0.0, 1.0),
              ("t_clamped", 2.5, 0.0, 1.0), ("t_interior", 0.3, 0.0, 1.0), ("d_at_eps", 4e-7, 0.0, EPS_D),
              ("d_below_eps", 4e-7, 0.0, below), ("d_above_eps", 4e-7, 0.0, above), ("d_negative", 0.25, 1.0, 0.0),
              ("t_negative_zero", 1.0, 1.0, 0.0), ("time_eq_stop", 0.5, 0.5, 0.5),
              ("time_below_stop", np.nextafter(F(0.5), F(0)), 0.5, 0.5), ("t_subnormal", 1e-10, 0.0, 1e30)]
    for k, (cls, time, t0, t1) in enumerate(factor):
        out.append(_case(f"{cls}_{k}", cls, time, t0, t1, base_l, base_r))
    out.append(_case("lanes", "lanes", 0.3, 0.0, 1.0, base_l, base_r))
    out.append(_case("lanes_t_zero", "lanes_t_zero", 0.0, 0.0, 1.0, base_l, base_r))
    out.append(_case("same", "same", 0.3, 0.0, 1.0, base_l, base_r, same=True))
    ql, qr = _quaternion_specials(13)
    out.append(_case("quaternions", "quaternions", 0.5, 0.0, 1.0, _concat(probe_l, ql, fl), _concat(probe_r, qr, fr)))
    hl, hr = _fill(64, 17)
    out.append(_case("f16_halves", "f16_halves", 0.5, 0.0, 1.0, _concat(probe_l, hl, fl), _concat(probe_r, hr, fr),
                     halves=True, seed=17))
    return out
