"""Clouds built splat by splat to pin the blend stage's coverage decisions (csrc/raster.cu) against the oracle.

Two kinds of frame:

* **Saturated frames.**  Every splat has opacity * global_opacity = 16384, so every covered pixel's alpha is the
  0.999 clamp (USE_OBB: exp(-4.5 |uv|^2) >= exp(-9) and 16384 exp(-9) = 2.0; USE_AABB: adaptive radius off and
  near-isotropic splats, so the quad's corner power stays near -9 too).  One covering splat leaves T = 1 - 0.999f and two
  leave T < T_STOP, both exact in f32 whichever way T is updated, so each pixel is 0.999 c1 + 0.000999 c2 of its first two
  covering splats and a GPU frame can be held to a few ulps of the oracle's f32 frame: a coverage map.
* **Knife-edge frames.**  Splats whose coverage of one target pixel turns on the last ulp: the deciding quantity (OBB
  max(|u|, |v|) against 1; AABB max(|mx|, |my|) against Rq) is found by walking the splat's scale one f32 ulp at a time
  (u and Rq move with 1 / scale and scale) and probing each candidate with the oracle.  The knife splats are the
  nearest ones and lie apart, so each is the first blended splat at its pixel when it covers it; behind them is a
  background of ordinary splats.

Classes of (splat, pixel) pairs a frame reaches (`pair_classes`):
  K0 / K+ / K-   the deciding quantity is exactly the threshold / one ulp above (not covered) / one ulp below
  KF             the decision differs when u, v are a rounded multiply plus a rounded add instead of the fma
  KS             the pixel is a corner pixel of its warp's 8x4 rectangle, the splat's centre lies outside that
                 rectangle diagonally and the decision is within 4 ulps: the separating-axis cull of raster_kernel<0>
                 decides on its slack
  KCH0 / KCH1    the pair sits in chunk 0 / chunk >= 1 of a tile with more than 256 entries (the TMA double buffer)
  KPOS_EVEN / KPOS_ODD / KPOS_TAIL   raster_kernel<0, false>: the splat's position in its warp's candidate list
                 (first or second of a pair, or the last of an odd-length list)
  KF_EVEN / KF_ODD / KF_TAIL   KF pairs at each of those positions (each has its own copy of the u, v arithmetic)
  KPX0 / KPX1    raster2_kernel: the pixel is its lane's first / second pixel

A pair far outside the frame (centre 1e4 px away) cannot be built: key-gen culls every centre beyond |ndc| = 1.1,
i.e. more than 0.05 W px outside the frame.
"""
from __future__ import annotations

import dataclasses
import functools

import numpy as np

import bevy_gaussian_splatting_b200 as B

SHC0 = 0.28209479177387814
SAT_OPACITY, SAT_GLOBAL = 16.0, 1024.0        # opacity * global_opacity = 16384
SAT_GLOBAL_2D_AABB = 2.0 ** 26                # surfel quads reach power -16 .. -20 at their corners: 16 * 2^26 e^-20.5 > 0.999
RT_CHUNK = 256
ROUND_FRACS = (16, 128, 1024, 8192)           # api.cu CHUNK_FRAC: inner round boundaries, in 1/65536 of n_visible

# geometry name -> (gaussian_mode, aabb)
GEOMETRIES = {"obb3d": (B.GaussianMode.Gaussian3d, False), "aabb3d": (B.GaussianMode.Gaussian3d, True),
              "aabb2d": (B.GaussianMode.Gaussian2d, True), "obb2d": (B.GaussianMode.Gaussian2d, False)}


def settings_for(geom: str, saturated: bool, **kw) -> B.CloudSettings:
    gm, aabb = GEOMETRIES[geom]
    base = dict(gaussian_mode=gm, aabb=aabb, color_space=B.GaussianColorSpace.LinRec709Display,
                opacity_adaptive_radius=not aabb, global_scale=1.0, binning_rounds=False)
    if saturated:
        base["global_opacity"] = SAT_GLOBAL_2D_AABB if geom == "aabb2d" else SAT_GLOBAL
    base.update(kw)
    return B.CloudSettings(**base)


def colours(n: int, seed: int, lo: float = 0.1, hi: float = 0.9) -> np.ndarray:
    """Per-splat linear colours in [lo, hi]: three low-discrepancy sequences, so that splats of nearby indices differ
    in some channel.  Knife splats take [0.7, 0.95] and the background behind them [0.1, 0.55]: every channel of a knife
    splat differs from what lies behind it by >= 0.15."""
    k = np.arange(n, dtype=np.float64) + seed * 7.0
    f = np.stack([(k * 0.6180339887) % 1.0, (k * 0.4142135624 + 0.3) % 1.0, (k * 0.7320508076 + 0.6) % 1.0], 1)
    return (lo + (hi - lo) * f).astype(np.float32)


class Splats:
    """Screen-space description -> a PlanarGaussian3d.  Each splat is flat and faces the camera of `view`: its screen
    covariance is its xy covariance times (focal / depth)^2 plus the 0.3 px^2 blur; it is turned about the view axis by
    `theta` (screen angle of its first axis is -theta)."""

    def __init__(self, view):
        self.view = view
        self.W, self.H = float(view.width), float(view.height)
        self.f = float(view.clip_from_view[1, 1])

    def depth(self, cx, cy, dist):
        a = (cx - self.W / 2) / (self.f * self.H / 2)
        b = (self.H / 2 - cy) / (self.f * self.H / 2)
        t = dist / np.sqrt(1 + a * a + b * b)
        return a, b, t

    def scale_for(self, half_px, t, cutoff):
        """World scale whose quad half-extent along that axis is `half_px` pixels at view depth t."""
        return t / (self.f * self.H) * np.sqrt(np.maximum((2.0 * np.asarray(half_px) / cutoff) ** 2 - 0.3, 1e-6))

    def cloud(self, cx, cy, dist, sa, sb, theta, opacity, rgb):
        cx, cy, dist, sa, sb, theta, opacity = (np.broadcast_to(np.asarray(v, np.float64), np.shape(cx))
                                                for v in (cx, cy, dist, sa, sb, theta, opacity))
        n = len(cx)
        a, b, t = self.depth(cx, cy, dist)
        pos = np.stack([a * t, 1.5 + b * t, 5.0 - t, np.ones(n)], 1)
        rot = np.stack([np.cos(theta / 2), np.zeros(n), np.zeros(n), np.sin(theta / 2)], 1)
        so = np.stack([sa, sb, 1e-3 * np.minimum(sa, sb), opacity], 1)
        sh = np.zeros((n, 48), np.float32)
        sh[:, :3] = (np.asarray(rgb, np.float64) - 0.5) / SHC0     # higher bands zero: colour = 0.5 + SHC0 dc
        return B.PlanarGaussian3d(pos.astype(np.float32), sh, rot.astype(np.float32), so.astype(np.float32))


def concat(*clouds):
    return B.PlanarGaussian3d(*(np.concatenate([getattr(c, k) for c in clouds]) for k in
                                ("position_visibility", "spherical_harmonic", "rotation", "scale_opacity")))


def cutoff_of(s: B.CloudSettings, opacity: float) -> float:
    return float(np.sqrt(max(9.0 + 2.0 * np.log(opacity), 1e-6))) if s.opacity_adaptive_radius else 3.0


# ---------------------------------------------------------------------------------------------------------------------
# saturated frames

@functools.lru_cache(maxsize=None)
def saturated_case(geom: str, n: int = 1500, w: int = 256, h: int = 192, seed: int = 0):
    """n splats of 2..14 px half-extent scattered over the frame at opacity * global_opacity = 16384.  USE_OBB splats
    take any orientation and aspects up to 2.5; USE_AABB ones are near-isotropic."""
    view = B.headless_view(w, h)
    s = settings_for(geom, saturated=True)
    rng = np.random.default_rng(1000 + seed + 17 * list(GEOMETRIES).index(geom))
    sp = Splats(view)
    cx, cy = rng.uniform(-4, w + 4, n), rng.uniform(-4, h + 4, n)
    dist = np.sort(rng.uniform(3.0, 30.0, n))
    _, _, t = sp.depth(cx, cy, dist)
    r = rng.uniform(2.0, 14.0, n)
    aniso = rng.uniform(1.0, 2.5, n) if not GEOMETRIES[geom][1] else rng.uniform(1.0, 1.02, n)
    theta = rng.uniform(-np.pi, np.pi, n)
    c = cutoff_of(s, SAT_OPACITY)
    cloud = sp.cloud(cx, cy, dist, sp.scale_for(r, t, c), sp.scale_for(r / aniso, t, c), theta, SAT_OPACITY,
                     colours(n, seed))
    return cloud, view, s


# ---------------------------------------------------------------------------------------------------------------------
# knife-edge frames

@dataclasses.dataclass
class KnifeCase:
    cloud: B.PlanarGaussian3d
    view: object
    settings: B.CloudSettings
    knife_ids: np.ndarray          # cloud index of each knife splat
    pixels: np.ndarray             # (k, 2) int target pixel of each


def _probe_at(oracle, cloud, view, s, ids, pix):
    u = B.GaussianSplattingPlugin.cloud_uniform(s)
    rec = oracle.project(cloud, view.to_abi(), u, s.to_abi(), ids)
    return rec, oracle.coverage_probe(rec, s.to_abi(), pix.astype(np.float32) + 0.5)


def deciding(probe, aabb: bool):
    """-> (quantity, threshold) as f32: the pair is covered iff quantity <= threshold (and the other test passes)."""
    if aabb:
        return np.maximum(np.abs(probe["mx"]), np.abs(probe["my"])), probe["Rq"]
    return np.maximum(np.abs(probe["u"]), np.abs(probe["v"])), np.ones(len(probe), np.float32)


def ulps_from(q, thr):
    """Signed distance of f32 q from f32 thr in ulps (positive: q above thr)."""
    def ordinal(x):
        b = np.asarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(b < 0, -(b & 0x7FFFFFFF), b)
    return ordinal(q) - ordinal(thr)


WALK = 160         # candidates each side of the fitted scale


def knife_case(oracle, geom: str, saturated: bool, n_knife: int = 96, w: int = 384, h: int = 256, seed: int = 0,
               blockers: int = 3, heavy: bool = False) -> KnifeCase:
    """`n_knife` knife splats on target pixels 32 px apart (half of them corner pixels of their warp's 8x4 rectangle
    with the splat's centre outside it diagonally), nearest to the camera; `blockers` tiles get 300 one-pixel splats in
    front of their knife splat (away from its pixel) so that its pair lands in the tile's second chunk; behind them a
    background of splats (`heavy`: big ones, so that the frame has >= 8 pairs per visible splat).  Unless `heavy`, the
    background keeps out of the warp rectangles of every fourth knife splat with 0 or 2 front dots: there the knife
    splat ends an odd-length candidate list (raster_kernel<0, false>'s odd tail), and it takes a fused/unfused split
    where its scale walk meets one."""
    gm, aabb = GEOMETRIES[geom]
    s = settings_for(geom, saturated)
    op = SAT_OPACITY if saturated else 0.9
    rng = np.random.default_rng(5000 + seed + 31 * list(GEOMETRIES).index(geom) + (7 if saturated else 0))
    view = B.headless_view(w, h)
    sp = Splats(view)
    # target pixels: one per 32 x 32 cell, away from the frame edge
    gx, gy = np.meshgrid(np.arange(16, w - 16, 32), np.arange(16, h - 16, 32))
    cells = np.stack([gx.ravel(), gy.ravel()], 1)
    cells = cells[rng.permutation(len(cells))[:n_knife]]
    k = len(cells)
    corner = np.arange(k) % 2 == 0
    pix = cells.copy()
    # corner pixels: snap to a warp-rectangle corner (x: wx0 or wx0 + 7, y: wy0 or wy0 + 3)
    sx, sy = rng.integers(0, 2, k), rng.integers(0, 2, k)
    pix[corner, 0] = (pix[corner, 0] // 8) * 8 + 7 * sx[corner]
    pix[corner, 1] = (pix[corner, 1] // 4) * 4 + 3 * sy[corner]
    # direction from the pixel to the splat centre: outward-diagonal for corner pixels, any for the rest
    phi = rng.uniform(-np.pi, np.pi, k)
    ddx = np.where(sx == 1, 1.0, -1.0) * rng.uniform(0.3, 1.0, k)
    ddy = np.where(sy == 1, 1.0, -1.0) * rng.uniform(0.3, 1.0, k)
    phi[corner] = np.arctan2(ddy[corner], ddx[corner])
    dist_px = rng.uniform(4.0, 9.0, k)
    cx = pix[:, 0] + 0.5 + dist_px * np.cos(phi)
    cy = pix[:, 1] + 0.5 + dist_px * np.sin(phi)
    theta = -phi                                    # first axis along the pixel -> centre direction
    dist = rng.uniform(3.0, 4.0, k)
    _, _, t = sp.depth(cx, cy, dist)
    c = cutoff_of(s, op)
    major = dist_px if not aabb else dist_px * np.maximum(np.abs(np.cos(phi)), np.abs(np.sin(phi)))
    aniso = rng.uniform(1.3, 2.0, k) if not aabb else np.ones(k)
    sa, sb = sp.scale_for(major, t, c), sp.scale_for(major / aniso, t, c)
    if aabb:
        sb = sa * rng.uniform(0.995, 1.0, k)
        theta = rng.uniform(0.1, 0.5, k)
    rgb = colours(k, seed, 0.7, 0.95)
    ids = np.arange(k, dtype=np.uint32)
    nf = np.arange(k) % 3                                   # front dots of each knife splat (below)
    tail = np.flatnonzero((np.arange(k) >= 2 * blockers) & (nf != 1) & (np.arange(k) % 4 == 3)) if not heavy else []
    # fit: u (OBB) ~ 1 / extent, Rq (AABB) ~ extent; a few f64 corrections, then an f32-ulp walk of both scales
    blur = 0.3 if gm == B.GaussianMode.Gaussian3d else 0.0       # (surfels get no screen-space blur)
    for _ in range(8):
        cl = sp.cloud(cx, cy, dist, sa, sb, theta, op, rgb)
        _, pr = _probe_at(oracle, cl, view, s, ids, pix)
        q, thr = deciding(pr, aabb)
        ratio = (q / thr).astype(np.float64)
        ratio = np.where(np.isfinite(ratio) & (ratio > 0.2) & (ratio < 5), ratio, 1.0)
        # extent^2 ~ sigma^2 + 0.3; OBB u ~ 1 / extent and AABB Rq ~ extent, so q / threshold = 1 wants the extent
        # times that ratio in both cases
        for arr in (sa, sb):
            sig2 = (arr * sp.f * sp.H / t) ** 2
            new = (sig2 + blur) * ratio ** 2 - blur
            arr[:] = t / (sp.f * sp.H) * np.sqrt(np.maximum(new, 1e-6))
    steps = np.arange(-WALK, WALK + 1)
    sa32, sb32 = sa.astype(np.float32), sb.astype(np.float32)
    cand_sa = (sa32.view(np.int32)[:, None] + steps[None, :]).astype(np.int32).view(np.float32)
    cand_sb = (sb32.view(np.int32)[:, None] + steps[None, :]).astype(np.int32).view(np.float32)
    rep = lambda a: np.repeat(np.asarray(a), len(steps))
    cl = sp.cloud(rep(cx), rep(cy), rep(dist), cand_sa.ravel().astype(np.float64), cand_sb.ravel().astype(np.float64),
                  rep(theta), op, np.repeat(rgb, len(steps), 0))
    # (float64 -> float32 in `cloud` is exact: the candidates are f32 values)
    _, pr = _probe_at(oracle, cl, view, s, np.arange(len(cl), dtype=np.uint32), np.repeat(pix, len(steps), 0))
    q, thr = deciding(pr, aabb)
    du = ulps_from(q, thr).reshape(k, len(steps))
    fused_diff = (pr["covered"] != pr["covered_if_unfused"]).reshape(k, len(steps))
    want = np.array([0, 1, -1])[np.arange(k) % 3]          # K0, K+, K-
    pick = np.empty(k, np.int64)
    for i in range(k):
        fd = np.flatnonzero(fused_diff[i])
        hit = np.flatnonzero(du[i] == want[i])
        if (i % 4 == 1 or i in tail) and len(fd):         # every fourth splat and the tail ones: prefer a fused/unfused split
            pick[i] = fd[len(fd) // 2]
        elif len(hit):
            pick[i] = hit[len(hit) // 2]
        else:
            pick[i] = int(np.argmin(np.abs(du[i] - want[i])))
    sel = np.arange(k) * len(steps) + pick
    sa_f, sb_f = cand_sa.ravel()[sel], cand_sb.ravel()[sel]
    knife = sp.cloud(cx, cy, dist, sa_f.astype(np.float64), sb_f.astype(np.float64), theta, op, rgb)
    parts = [knife]
    nb = 0

    def dots(xy, d, cseed):
        # one-pixel splats (quad half-extent 0.9 px; surfels 2 px: a smaller surfel quad is its 0.707 cutoff floor, whose
        # corners a saturated opacity no longer saturates) centred on the given pixels at distances d
        _, _, bt = sp.depth(xy[:, 0] + 0.5, xy[:, 1] + 0.5, d)
        bs = sp.scale_for(np.full(len(xy), 0.9 if blur else 2.0), bt, cutoff_of(s, op))
        return sp.cloud(xy[:, 0] + 0.5, xy[:, 1] + 0.5, d, bs, bs * 0.999, 0.3, op, colours(len(xy), cseed, 0.1, 0.55))

    # blockers: 300 one-pixel splats in the knife splat's tile, at least 5 px from its pixel: in front of it in the
    # first `blockers` tiles (its pair lands in chunk 1), behind it in the next `blockers` ones (chunk 0 of a TMA tile)
    for i in range(min(2 * blockers, k)):
        tx, ty = (pix[i] // 16) * 16
        bx, by = np.meshgrid(np.arange(tx, tx + 16), np.arange(ty, ty + 16))
        far = (np.abs(bx - pix[i, 0]) >= 5) | (np.abs(by - pix[i, 1]) >= 5)
        bxy = np.stack([bx[far], by[far]], 1)
        bxy = bxy[rng.integers(0, len(bxy), 300)]
        front = i < blockers
        parts.insert(0, dots(bxy, rng.uniform(1.5, 2.5, 300) if front else rng.uniform(5.0, 7.0, 300), seed + 50 + i))
        nb += 300
    # fronts: 0, 1 or 2 one-pixel splats nearer than the knife splat in its warp's 8x4 rectangle, >= 4 px from its
    # pixel, so that it sits at an even or odd position of that warp's candidate list
    fxy = []
    for i in np.flatnonzero(nf):
        wx0, wy0 = (pix[i, 0] // 8) * 8, (pix[i, 1] // 4) * 4
        fx = wx0 + (0 if pix[i, 0] - wx0 >= 4 else 7)
        for _ in range(nf[i]):
            fxy.append((fx, wy0 + int(rng.integers(0, 4))))
    if fxy:
        parts.insert(0, dots(np.asarray(fxy, np.float64), rng.uniform(2.6, 2.9, len(fxy)), seed + 77))
        nb += len(fxy)
    # background
    nbg = 1500 if not heavy else 600
    bcx, bcy = rng.uniform(0, w, nbg), rng.uniform(0, h, nbg)
    bdist = rng.uniform(8.0, 30.0, nbg)
    _, _, bt = sp.depth(bcx, bcy, bdist)
    br = rng.uniform(3.0, 12.0, nbg) if not heavy else rng.uniform(24.0, 60.0, nbg)
    bani = rng.uniform(1.0, 2.0, nbg) if not aabb else np.ones(nbg)
    bop = op if saturated else rng.uniform(0.3, 0.95, nbg)
    cb = cutoff_of(s, 0.6 if not saturated else op)
    bg = sp.cloud(bcx, bcy, bdist, sp.scale_for(br, bt, cb), sp.scale_for(br / bani, bt, cb) * 0.999,
                  rng.uniform(-np.pi, np.pi, nbg), bop, colours(nbg, seed + 99, 0.1, 0.55))
    if not heavy:
        w0 = (pix[tail] // [8, 4]) * [8, 4]
        rec = oracle.project(bg, view.to_abi(), B.GaussianSplattingPlugin.cloud_uniform(s), s.to_abi(),
                             np.arange(nbg, dtype=np.uint32))
        hits = ((rec["xlo"][:, None] <= w0[None, :, 0] + 7) & (rec["xhi"][:, None] >= w0[None, :, 0]) &
                (rec["ylo"][:, None] <= w0[None, :, 1] + 3) & (rec["yhi"][:, None] >= w0[None, :, 1]))
        keep = ~hits.any(1)
        bg = B.PlanarGaussian3d(bg.position_visibility[keep], bg.spherical_harmonic[keep], bg.rotation[keep],
                                bg.scale_opacity[keep])
    parts.append(bg)
    cloud = concat(*parts)
    return KnifeCase(cloud, view, s, np.arange(nb, nb + k, dtype=np.uint32), pix)


def round_of(rank, n_vis):
    b = [(n_vis * f) >> 16 for f in ROUND_FRACS]
    return int(np.searchsorted(b, rank, side="right"))


def warp_candidates_r0(rec, tile_slice, chunk, wx0, wy0):
    """numpy replica of raster_kernel<0>'s per-warp candidate list for one chunk of a tile slice: bbox test, then the
    separating-axis test in f32 (same operations and order).  -> (list of ranks, ambiguous): `ambiguous` marks the
    ranks whose SAT value lies within 1e-4 relative of its threshold, where contraction by the compiler may decide."""
    f = np.float32
    ent = tile_slice[chunk * RT_CHUNK:(chunk + 1) * RT_CHUNK]
    r = rec[ent]
    tile_x, tile_y = wx0 // 16, wy0 // 16
    tcx, tcy = f(tile_x * 16 + 8), f(tile_y * 16 + 8)
    rcx, rcy = f(wx0 + 4), f(wy0 + 2)
    hit = ~((r["xhi"] < wx0) | (r["xlo"] > wx0 + 7) | (r["yhi"] < wy0) | (r["ylo"] > wy0 + 3))
    cx, cy, ux, uy, vx, vy = (r[k].astype(f) for k in ("cx", "cy", "ux", "uy", "vx", "vy"))
    ax = np.abs(cx - tcx) + f(4)
    ay = np.abs(cy - tcy) + f(6)
    ur = np.abs(ux) * f(3.5) + np.abs(uy) * f(1.5)
    vr = np.abs(vx) * f(3.5) + np.abs(vy) * f(1.5)
    um = np.abs(ux) * ax + np.abs(uy) * ay + ur
    vm = np.abs(vx) * ax + np.abs(vy) * ay + vr
    thx = ur + f(1) + f(1e-5) * um
    thy = vr + f(1) + f(1e-5) * vm
    dxc, dyc = rcx - cx, rcy - cy
    sx_ = np.abs(ux * dxc + uy * dyc)
    sy_ = np.abs(vx * dxc + vy * dyc)
    with np.errstate(invalid="ignore"):
        cull = (sx_ > thx) | (sy_ > thy)
        amb = (np.abs(sx_ - thx) <= 1e-4 * thx) | (np.abs(sy_ - thy) <= 1e-4 * thy)
    keep = hit & ~cull
    return ent[keep], set(ent[hit & amb].tolist())


def pair_classes(oracle, case: KnifeCase, til=None, trace=None):
    """-> dict class -> list of knife indices, plus per-knife info.  Only pairs whose decision is visible in the frame
    count: a covered knife splat must be the first blended splat at its pixel, an uncovered one must have no nearer
    splat blended there."""
    s, view = case.settings, case.view
    aabb = bool(s.aabb)
    u = B.GaussianSplattingPlugin.cloud_uniform(s)
    if til is None:
        til = oracle.render_tiles(case.cloud, view.to_abi(), u, s.to_abi(), want_image=False)
    if trace is None:
        trace = oracle.blend_trace(case.cloud, view.to_abi(), u, s.to_abi())
    r2i = til["rank_to_id"]
    id2rank = np.full(len(case.cloud), -1, np.int64)
    id2rank[r2i] = np.arange(len(r2i))
    rec = oracle.project(case.cloud, view.to_abi(), u, s.to_abi(), r2i)
    ranks = id2rank[case.knife_ids]
    pix = case.pixels
    pr = oracle.coverage_probe(rec[np.maximum(ranks, 0)], s.to_abi(), pix.astype(np.float32) + 0.5)
    q, thr = deciding(pr, aabb)
    du = ulps_from(q, thr)
    W = view.width
    tiles_x = -(-W // 16)
    out = {k: [] for k in ("K0", "K+", "K-", "KF", "KS", "KCH0", "KCH1", "KPOS_EVEN", "KPOS_ODD", "KPOS_TAIL",
                           "KPX0", "KPX1", "ROUND_GE1")}
    visible = np.zeros(len(ranks), bool)
    n_vis = til["n_vis"]
    for i, (rk, (x, y)) in enumerate(zip(ranks, pix)):
        if rk < 0:
            continue
        tr = trace[y, x]
        cov = bool(pr["covered"][i])
        vis = (tr["rank0"] == rk) if cov else (tr["rank0"] == -1 or tr["rank0"] > rk)
        if not vis:
            continue
        visible[i] = True
        if du[i] == 0:
            out["K0"].append(i)
        elif du[i] == 1:
            out["K+"].append(i)
        elif du[i] == -1:
            out["K-"].append(i)
        if pr["covered"][i] != pr["covered_if_unfused"][i]:
            out["KF"].append(i)
        wx0, wy0 = (x // 8) * 8, (y // 4) * 4
        r = rec[rk]
        corner = x in (wx0, wx0 + 7) and y in (wy0, wy0 + 3)
        outside_diag = (r["cx"] < wx0 or r["cx"] > wx0 + 8) and (r["cy"] < wy0 or r["cy"] > wy0 + 4)
        if corner and outside_diag and abs(int(du[i])) <= 4:
            out["KS"].append(i)
        t = (y // 16) * tiles_x + x // 16
        a, b = til["tile_ranges"][t]
        sl = til["tile_entries"][a:b]
        pos = int(np.flatnonzero(sl == rk)[0])
        if b - a > RT_CHUNK:
            out["KCH0" if pos < RT_CHUNK else "KCH1"].append(i)
        if not aabb:
            lst, amb = warp_candidates_r0(rec, sl, pos // RT_CHUNK, wx0, wy0)
            if rk not in amb:
                li = np.flatnonzero(lst == rk)
                if len(li):
                    j = int(li[0])
                    if j == len(lst) - 1 and len(lst) % 2 == 1:
                        out["KPOS_TAIL"].append(i)
                    else:
                        out["KPOS_EVEN" if j % 2 == 0 else "KPOS_ODD"].append(i)
            out["KPX0" if x % 2 == 0 else "KPX1"].append(i)
        if round_of(rk, n_vis) >= 1:
            out["ROUND_GE1"].append(i)
    for pos in ("EVEN", "ODD", "TAIL"):       # fma splits at each position: each has its own copy of the u, v arithmetic
        out["KF_" + pos] = sorted(set(out["KF"]) & set(out["KPOS_" + pos]))
    return out, dict(ranks=ranks, du=du, visible=visible, probe=pr, rec=rec, til=til, trace=trace)


# ---------------------------------------------------------------------------------------------------------------------
# the per-pixel error bound of a kernel's blend against the float64 evaluation of the same walk

U = 2.0 ** -24                 # unit roundoff of f32
T_STOP = 1e-4


def alpha_error_coefs(aabb: bool):
    """(c0, c1): the kernel's blended alpha a = min(e * o, 0.999) is within (c0 + c1 |p|) U relative of the oracle's
    min(exp(p) * o, 0.999) with exp in f64 of the f32 power p.
    USE_OBB (ex2.approx.ftz.f32 of qd * -6.492127684f): the constant and the product are each rounded (2 U |p| log2 e in
    the exponent, i.e. 2 U |p| relative on e), the oracle's power -4.5 qd is rounded (U |p|), ex2.approx is within 2 ulp
    (4 U), and e * o is rounded on both sides (2 U): (6 + 3 |p|) U.
    USE_AABB (__expf of the same f32 power on both sides): __expf is within 2 + floor(1.173 |p|) ulp, i.e.
    (4 + 2.35 |p|) U relative, plus the two roundings of e * o: (6 + 2.35 |p|) U."""
    return (6.0, 2.35) if aabb else (6.0, 3.0)


def blend_bounds(trace, aabb: bool, dc: float = 0.0):
    """-> (bound on |C - c64| per channel, bound on |T - T64|, near_stop mask) per pixel.

    With da_j the alpha error above, n the blended count and m = max |c| of the blended records:
    * alpha errors: moving a_j by da changes w_j = a_j T_j by da T_j and scales every later weight by (1 - a_j - da) /
      (1 - a_j), whose total is <= T_j (1 - a_j); so |dC| <= 2 m sum_j |da_j| T_j = 2 m U (c0 (1 - T64) + c1 w_power)
      (w_power = sum w_j |p_j|), and |dT| / T <= sum_j |da_j| / (1 - a_j) = U (c0 t_sens + c1 t_sens_power) (sums of
      a / (1 - a) and a |p| / (1 - a) over the alphas below the clamp: a clamped alpha is 0.999 on both sides);
    * f32 rounding: w = a T (U), each fma into C (U m), each T update (U relative, so T_j is within j U): (2 n + 1) U m
      on C, (n + 1) U T on T;
    * record colours: the kernel's r, g, b differ from the oracle's by at most dc (rsqrt / __powf in the colour path),
      weighted by sum w = 1 - T: dc (1 - T64);
    * the stop: where some f32 T tested against T_STOP lies within the relative error of T of it, the kernel may stop
      one splat earlier or later than the oracle; the weight it adds or drops is <= T there ~ T_STOP: T_STOP m on C and
      T_STOP on T."""
    c0, c1 = alpha_error_coefs(aabb)
    n = trace["n_blended"].astype(np.float64)
    m = trace["max_c"].astype(np.float64)
    T64 = trace["T64"]
    t_rel = U * (c0 * trace["t_sens"] + c1 * trace["t_sens_power"]) + (n + 1) * U
    near_stop = (trace["n_blended"] > 0) & (trace["stop_margin"] <= np.maximum(1e-5, 2.0 * t_rel))
    da = U * (c0 * (1.0 - T64) + c1 * trace["w_power"])
    bc = m * (2.0 * da + (2.0 * n + 1.0) * U) + dc * (1.0 - T64) + np.where(near_stop, 1.01 * T_STOP * m, 0.0)
    bt = T64 * t_rel + np.where(near_stop, 1.01 * T_STOP, 0.0)
    return bc, bt, near_stop


def expected_frame(trace, out_mode: str, dst=None):
    """(H, W, 4) float64 frame from the trace: opaque (C, 1), premultiplied (C, 1 - T), over (C + T dst.rgb,
    (1 - T) + T dst.a)."""
    C, T = trace["c64"], trace["T64"][..., None]
    if out_mode == "opaque":
        return np.concatenate([C, np.ones_like(T)], -1)
    if out_mode == "premultiplied":
        return np.concatenate([C, 1.0 - T], -1)
    d = dst.astype(np.float64)
    return np.concatenate([C + T * d[..., :3], (1.0 - T) + T * d[..., 3:4]], -1)


def frame_bounds(trace, aabb: bool, out_mode: str, dc: float = 0.0, dst=None):
    """(H, W, 4) bound on |frame - expected_frame| (f32 output), and the near-stop mask."""
    bc, bt, ns = blend_bounds(trace, aabb, dc)
    bc, bt = bc[..., None], bt[..., None]
    if out_mode == "opaque":
        b = np.concatenate([np.repeat(bc, 3, -1), np.zeros_like(bt)], -1)
    elif out_mode == "premultiplied":
        b = np.concatenate([np.repeat(bc, 3, -1), bt + U], -1)
    else:
        d = np.abs(dst.astype(np.float64))
        b = np.concatenate([bc + bt * d[..., :3] + 2 * U * (np.abs(trace["c64"]) + d[..., :3]), bt * (1.0 + d[..., 3:4]) + 3 * U], -1)
    return b, ns
