"""Gaussian4d cases and the numpy restatement of bgs_render_4d's rule (include/bgs.h), independent of the C++ oracle:
the fixed-series exp and cos, the conditioning on time and Velocity, every step an f32 numpy operation (numpy rounds
each one and never fuses) in the order the header writes it.  Used by tests/test_oracle_temporal.py (against
temporal_oracle/) and tests/test_gpu_temporal.py (case clouds)."""
from __future__ import annotations

import numpy as np

import bevy_gaussian_splatting_b200 as B

f32 = np.float32


def det_exp(x) -> np.ndarray:
    x = np.asarray(x, np.float32)
    out = np.empty(x.shape, np.float32)
    for i, xf in np.ndenumerate(x):
        if np.isnan(xf):
            out[i] = xf
            continue
        if xf < f32(-110.0):
            out[i] = 0.0
            continue
        if xf > f32(89.0):
            out[i] = np.inf
            continue
        xd = float(xf)
        k = float(np.rint(xd * 1.4426950408889634))
        r = xd - k * 0.6931471805599453
        c = [1.0]
        for j in range(1, 17):
            c.append(c[-1] / float(j))
        p = c[16]
        for j in range(15, -1, -1):
            p = p * r + c[j]
        with np.errstate(over="ignore"):
            out[i] = np.float32(p * 2.0 ** int(k))
    return out


def det_cos(x) -> np.ndarray:
    x = np.asarray(x, np.float32)
    out = np.empty(x.shape, np.float32)
    for i, xf in np.ndenumerate(x):
        if not np.isfinite(xf):
            out[i] = np.nan
            continue
        xd = float(xf)
        k = float(np.rint(xd * 0.15915494309189535))
        r = xd - k * 6.283185307179586
        z = r * r
        c = [1.0]
        for j in range(1, 19):
            c.append(-c[-1] / float((2 * j - 1) * (2 * j)))
        p = c[18]
        for j in range(17, -1, -1):
            p = p * z + c[j]
        out[i] = np.float32(p)
    return out


def condition(rot8, so, tt, gs, t):
    """-> (cov6 (n, 6), delta_mean (n, 3), marginal (n,), mask (n,)), include/bgs.h's steps 3-5."""
    rot8, so, tt = (np.asarray(a, np.float32).reshape(-1, w) for a, w in ((rot8, 8), (so, 4), (tt, 4)))
    gs, t = f32(gs), f32(t)
    with np.errstate(all="ignore"):
        dt = t - tt[:, 0]
        sd = [gs * so[:, 0], gs * so[:, 1], gs * so[:, 2], tt[:, 1]]
        w, x, y, z, wr, xr, yr, zr = (rot8[:, i] for i in range(8))
        Ml = [[w, -x, -y, -z], [x, w, -z, y], [y, z, w, -x], [z, -y, x, w]]
        Mr = [[wr, -xr, -yr, -zr], [xr, wr, zr, -yr], [yr, -zr, wr, xr], [zr, yr, -xr, wr]]
        R = [[((Mr[0][r] * Ml[c][0] + Mr[1][r] * Ml[c][1]) + Mr[2][r] * Ml[c][2]) + Mr[3][r] * Ml[c][3] for r in range(4)]
             for c in range(4)]
        M = [[R[c][r] * sd[c] for r in range(4)] for c in range(4)]
        S = [[((M[r][0] * M[c][0] + M[r][1] * M[c][1]) + M[r][2] * M[c][2]) + M[r][3] * M[c][3] for r in range(4)]
             for c in range(4)]
        cov_t = S[3][3]
        marginal = det_exp(((f32(-0.5) * dt) * dt) / cov_t)
        mask = marginal > f32(0.05)
        c12 = [S[0][3], S[1][3], S[2][3]]
        cond = lambda c, r: S[c][r] - (c12[c] * c12[r]) / cov_t  # noqa: E731
        cov6 = np.stack([cond(0, 0), cond(0, 1), cond(0, 2), cond(1, 1), cond(1, 2), cond(2, 2)], 1).astype(np.float32)
        dm = np.stack([(c12[i] / cov_t) * dt for i in range(3)], 1).astype(np.float32)
    cov6[~mask] = 0.0
    dm[~mask] = 0.0
    return cov6, dm, marginal, mask


def velocity(rot8, so, tt, gs, t):
    """-> (rgb (n, 3), zero_opacity (n,)): Velocity's colour (include/bgs.h, 7.) of every masked-in gaussian."""
    _, dm, _, _ = condition(rot8, so, tt, gs, t)
    _, fdm, _, _ = condition(rot8, so, tt, gs, f32(t) + f32(1e-3))   # (a failed mask's delta_mean is 0)
    with np.errstate(all="ignore"):
        v = (fdm - dm) / f32(1e-3)
        ln = np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])
        sc = np.fmin(np.fmax((ln - f32(1.0)) / (f32(2.0) - f32(1.0)), f32(0.0)), f32(1.0))
        zero = sc < f32(1e-2)
        rgb = ((f32(0.5) * (v / ln[:, None] + f32(1.0))) * sc[:, None]).astype(np.float32)
    rgb[zero] = 0.0
    return rgb, zero


def cloud_4d(pos, rot8=None, so=None, tt=None, sh=None, vis=None, seed=0) -> B.PlanarGaussian4d:
    """A PlanarGaussian4d at `pos` (n, 3); the rest seeded where not given."""
    pos = np.asarray(pos, np.float32).reshape(-1, 3)
    n = len(pos)
    base = B.random_gaussians_4d_seeded(n, seed)
    pv = np.concatenate([pos, np.ones((n, 1), np.float32) if vis is None else np.asarray(vis, np.float32).reshape(n, 1)], 1)
    return B.PlanarGaussian4d(pv, base.spherindrical_harmonic if sh is None else sh,
                              base.isotropic_rotations if rot8 is None else rot8,
                              base.scale_opacity if so is None else so, base.timestamp_timescale if tt is None else tt)


def scene_4d(n=4000, seed=0, spread=2.0, dist=0.0, selected=False) -> B.PlanarGaussian4d:
    """A seeded 4D cloud in front of `headless_view`'s camera (positions in a box of half-size `spread` around z =
    -dist, inside the view), timescales in [0.2, 1) so that some are masked
    at each time and some are not, visibility a mix of 0, 1 and class labels when `selected`."""
    c = B.random_gaussians_4d_seeded(n, seed)
    rng = np.random.default_rng(seed)
    pos = c.position_visibility.copy()
    pos[:, :3] = pos[:, :3] / f32(20.0) * f32(spread)
    pos[:, 2] -= f32(dist)
    if selected:
        pos[:, 3] = rng.choice(np.array([0.0, 1.0, 2.0, 3.5], np.float32), n)
    so = c.scale_opacity.copy()
    so[:, :3] *= f32(0.15)
    tt = c.timestamp_timescale.copy()
    tt[:, 1] = np.where(tt[:, 1] < 0, f32(-1.0), f32(1.0)) * (f32(0.2) + np.abs(tt[:, 1]) * f32(0.8))
    return B.PlanarGaussian4d(pos, c.spherindrical_harmonic * f32(0.3), c.isotropic_rotations, so, tt)


def fast_arrays(n=20000, seed=3):
    """(rot8, so, tt, t): gaussians whose Velocity is not 0.  transpose(M) * M of the reference's rule is diagonal up to
    rounding (R = M_r * M_l is a scaled 4D rotation), so space and time couple only through rounding: scales of 1e2 to
    1e6 over a timescale of 1e-3 make that coupling a velocity near 1, on both sides of scaled = 1e-2.  Some future
    masks fail.  t = timestamp + 1e-4."""
    c = B.random_gaussians_4d_seeded(n, seed)
    rng = np.random.default_rng(seed)
    so = c.scale_opacity.copy()
    so[:, :3] = (10 ** rng.uniform(2, 6, (n, 3))).astype(np.float32)
    tt = np.zeros((n, 4), np.float32)
    tt[:, 0], tt[:, 1] = 0.5, 1e-3
    return c.isotropic_rotations, so, tt, f32(0.5) + f32(1e-4)
