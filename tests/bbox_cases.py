"""Clouds built to pin the bounding-box overlay's edge decisions (BGS_FLAG_VISUALIZE_BOUNDING_BOX, include/bgs.h) against
the entity oracle, and the literal VISUALIZE_BOUNDING_BOX branch of the reference's fs_main (gaussian.wgsl:486-495).

Band-edge frames: like blend_cases.knife_case, but the pixel that decides is on the overlay's band edge instead of the
quad's.  Each knife splat's target pixel sits where s = uv * 0.5 + 0.5 of one axis (the one away from the splat's centre)
is within a few f32 ulps of 0.08f or 0.92f, or on it: the splat's scales are walked one ulp at a time and each candidate
is probed.  Half of the splats decide on s.x and half on s.y; the knife splats are the nearest ones and lie apart, so each
is the first blended splat at its pixel; behind them is a background of ordinary splats.
"""
from __future__ import annotations

import dataclasses

import numpy as np

import bevy_gaussian_splatting_b200 as B
import blend_cases as BC

F = np.float32
EDGE = F(0.08)
LO, HI = EDGE, F(F(1.0) - EDGE)
EDGE_RGB = np.array([0.3, 1.0, 0.1], np.float32)
BAND = 0.84          # |uv| of the band edge: s = 0.08 at uv = -0.84, 0.92 at +0.84
WALK = 160


def wgsl_visualize_bounding_box(uv_x, uv_y):
    """gaussian.wgsl:486-495, literally, in f32 (WGSL's f32 arithmetic is IEEE single; the multiply by 0.5 is exact):

        let uv = input.uv * 0.5 + 0.5;
        let edge_width = 0.08;
        if ((uv.x < edge_width || uv.x > 1.0 - edge_width) || (uv.y < edge_width || uv.y > 1.0 - edge_width)) {
            return vec4<f32>(0.3, 1.0, 0.1, 1.0);
        }

    -> (edge: bool array, s: (n, 2) the uv * 0.5 + 0.5 it tests).  The fragment colour of an edge is
    (0.3, 1.0, 0.1, 1.0): alpha exactly 1 under the premultiplied blend."""
    ux, uy = np.asarray(uv_x, F), np.asarray(uv_y, F)
    sx, sy = ux * F(0.5) + F(0.5), uy * F(0.5) + F(0.5)
    edge_width = F(0.08)
    edge = ((sx < edge_width) | (sx > F(1.0) - edge_width)) | ((sy < edge_width) | (sy > F(1.0) - edge_width))
    return edge, np.stack([sx, sy], -1)


def probe_uv(probe, aabb: bool):
    """The overlay's uv of coverage-probe pairs (oracle.coverage_probe): quad uv, or m / R (IEEE f32 division)."""
    if aabb:
        return probe["mx"] / probe["Rq"], probe["my"] / probe["Rq"]
    return probe["u"], probe["v"]


def deciding_s(s):
    """(s of the axis farther from 0.5, its band threshold) per pair."""
    ax = np.abs(s[:, 0] - F(0.5)) >= np.abs(s[:, 1] - F(0.5))
    sd = np.where(ax, s[:, 0], s[:, 1]).astype(F)
    return sd, np.where(sd < F(0.5), LO, HI).astype(F), ax


@dataclasses.dataclass
class BandCase:
    cloud: B.PlanarGaussian3d
    view: object
    settings: B.CloudSettings
    knife_ids: np.ndarray       # cloud index of each knife splat
    pixels: np.ndarray          # (k, 2) its target pixel
    ulps: np.ndarray            # signed f32 ulps of the deciding s from its band threshold
    on_x: np.ndarray            # the deciding axis is s.x


def band_case(oracle, geom: str, n_knife: int = 96, w: int = 384, h: int = 256, seed: int = 0, **settings) -> BandCase:
    gm, aabb = BC.GEOMETRIES[geom]
    s = dataclasses.replace(BC.settings_for(geom, False), **settings)
    op = 0.9
    rng = np.random.default_rng(7000 + seed + 31 * list(BC.GEOMETRIES).index(geom))
    view = B.headless_view(w, h)
    sp = BC.Splats(view)
    gx, gy = np.meshgrid(np.arange(16, w - 16, 32), np.arange(16, h - 16, 32))
    cells = np.stack([gx.ravel(), gy.ravel()], 1)
    pix = cells[rng.permutation(len(cells))[:n_knife]]
    k = len(pix)
    # direction pixel -> centre: quad-uv splats turn their major axis along it (theta = -phi) or their minor axis (every
    # other splat), so the deciding axis is u or v; conic and surfel quads are screen-aligned, so phi keeps near an axis
    if aabb:
        phi = (rng.integers(0, 4, k) * (np.pi / 2) + rng.uniform(-0.25, 0.25, k))
        theta = rng.uniform(0.1, 0.5, k)
    else:
        phi = rng.uniform(-np.pi, np.pi, k)
        theta = -phi + np.where(np.arange(k) % 2 == 1, np.pi / 2, 0.0)
    dist_px = rng.uniform(4.0, 8.0, k)
    cx = pix[:, 0] + 0.5 + dist_px * np.cos(phi)
    cy = pix[:, 1] + 0.5 + dist_px * np.sin(phi)
    dist = rng.uniform(3.0, 4.0, k)
    _, _, t = sp.depth(cx, cy, dist)
    c = BC.cutoff_of(s, op)
    major = dist_px / BAND if not aabb else dist_px * np.maximum(np.abs(np.cos(phi)), np.abs(np.sin(phi))) / BAND
    aniso = rng.uniform(1.2, 1.6, k) if not aabb else np.ones(k)
    sa = sp.scale_for(major, t, c)
    sb = sp.scale_for(major / aniso, t, c) if not aabb else sa * rng.uniform(0.995, 1.0, k)
    rgb = BC.colours(k, seed, 0.7, 0.95)
    ids = np.arange(k, dtype=np.uint32)
    blur = 0.3 if gm == B.GaussianMode.Gaussian3d else 0.0
    for _ in range(8):   # u ~ 1 / extent, m / R ~ 1 / extent: scale both extents by |uv| / BAND
        cl = sp.cloud(cx, cy, dist, sa, sb, theta, op, rgb)
        _, pr = BC._probe_at(oracle, cl, view, s, ids, pix)
        ux, uy = probe_uv(pr, aabb)
        ratio = (np.maximum(np.abs(ux), np.abs(uy)) / BAND).astype(np.float64)
        ratio = np.where(np.isfinite(ratio) & (ratio > 0.2) & (ratio < 5), ratio, 1.0)
        for arr in (sa, sb):
            sig2 = (arr * sp.f * sp.H / t) ** 2
            arr[:] = t / (sp.f * sp.H) * np.sqrt(np.maximum((sig2 + blur) * ratio ** 2 - blur, 1e-6))
    steps = np.arange(-WALK, WALK + 1)
    want = np.array([0, 1, -1, 2, -2, 4, -4])[np.arange(k) % 7]
    sa32, sb32 = sa.astype(F), sb.astype(F)
    rep = lambda a: np.repeat(np.asarray(a), len(steps))
    for _ in range(4):   # walk both scales one f32 ulp at a time around the best candidate so far
        cand_sa = (sa32.view(np.int32)[:, None] + steps[None, :]).astype(np.int32).view(F)
        cand_sb = (sb32.view(np.int32)[:, None] + steps[None, :]).astype(np.int32).view(F)
        cl = sp.cloud(rep(cx), rep(cy), rep(dist), cand_sa.ravel().astype(np.float64), cand_sb.ravel().astype(np.float64),
                      rep(theta), op, np.repeat(rgb, len(steps), 0))
        _, pr = BC._probe_at(oracle, cl, view, s, np.arange(len(cl), dtype=np.uint32), np.repeat(pix, len(steps), 0))
        _, sv = wgsl_visualize_bounding_box(*probe_uv(pr, aabb))
        sd, thr, ax = deciding_s(sv)
        du = BC.ulps_from(sd, thr)
        du = np.where(pr["covered"] != 0, du, 1 << 40).reshape(k, len(steps))
        pick = np.array([int(np.argmin(np.abs(du[i] - want[i]) * 1000 + np.abs(steps))) for i in range(k)])
        sel = np.arange(k) * len(steps) + pick
        sa32, sb32 = cand_sa.ravel()[sel], cand_sb.ravel()[sel]
        if (np.abs(du.reshape(-1)[sel] - want) <= 4).mean() > 0.9:
            break
    knife = sp.cloud(cx, cy, dist, sa32.astype(np.float64), sb32.astype(np.float64), theta, op, rgb)
    # background: ordinary splats behind the knife ones
    nbg = 1200
    bcx, bcy = rng.uniform(0, w, nbg), rng.uniform(0, h, nbg)
    bdist = rng.uniform(8.0, 30.0, nbg)
    _, _, bt = sp.depth(bcx, bcy, bdist)
    br = rng.uniform(3.0, 12.0, nbg)
    bani = rng.uniform(1.0, 2.0, nbg) if not aabb else np.ones(nbg)
    cb = BC.cutoff_of(s, 0.6)
    bg = sp.cloud(bcx, bcy, bdist, sp.scale_for(br, bt, cb), sp.scale_for(br / bani, bt, cb) * 0.999,
                  rng.uniform(-np.pi, np.pi, nbg), rng.uniform(0.3, 0.95, nbg), BC.colours(nbg, seed + 99, 0.1, 0.55))
    return BandCase(BC.concat(knife, bg), view, s, ids, pix, du.reshape(-1)[sel], ax[sel])
