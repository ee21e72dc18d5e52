"""Clouds built gaussian by gaussian to reach the branches and thresholds of the projection (csrc/project.cu,
`project_one` and the per-geometry and per-colour-source functions it dispatches to, `make_bbox`,
`depth_range_kernel`) and of key-gen's visibility and key (csrc/project_math.cuh: `keygen_world_pos`,
`in_frustum_fast`, `in_frustum`, `depth_key`).

Every case is a planar cloud with its view, its model transform, its layout (f32, f16, precomputed covariance) and
the settings it is meant for, plus `tags`: class name -> boolean mask over the cloud, counted with the oracle or with
a numpy f32 restatement of the deciding quantity in the oracle's own operation order.  Tests assert each class is
reached (`tests/test_oracle_project.py`) and hold the CUDA path to the oracle on every case
(`tests/test_gpu_project.py`).

Classes and what cannot be built exactly:

* DRAW_*: the visibility lane at 0.5 (Selected draws w >= 0.5, HighlightSelected highlights w > 0.5), its two f32
  neighbours, -0, negative, NaN, +-inf.
* CUT_*: f32 opacities around the `9 + 2 ln o > 1e-6` clamp.  Near o = e^-4.5 the sum 9 + 2 ln o is exact (Sterbenz)
  and a multiple of 2^-20, so it takes the values 0, 2^-20 = 9.54e-7 (clamped) and 2^-19 = 1.91e-6 (kept) but never
  1e-6f itself: `>` and `>=` there are the same function, and the knife is the last clamped / first kept opacity.
  Also o = 0, -0, negative, subnormal, NaN, inf and o > 1.
* SIG_*: Sigma = (S R)^T (S R) with entries zero, -0, subnormal, infinite or NaN under an identity model, where the
  projection's identity shortcut (`sigma3d`: T Sigma T^t == Sigma) must not be taken; SIG_SHORTCUT where it is, and SIG_SIGNZERO
  where the full product T Sigma T^t differs from Sigma in the sign of a zero.
* OBB quirks: EV_NAN (b = 0 and a = c: the NaN eigenvector, undrawn), B0_ANEC (b = +-0, a != c: l1 - a is 0 or one
  rounding from it), MINOR_NONFINITE ((a + c) - bb <= 0: the minor axis 0 or NaN, drawn with infinite v), and on the
  USE_AABB record DET_ZERO (det = 0: infinite conic, drawn) and DET_NAN (a * c overflows: NaN conic, drawn).
* BB_*: `make_bbox` edges whose ceil / floor argument is an integer (BB_ON), one ulp above (BB_UP) or below (BB_DOWN);
  within 1e-3 px of an integer on the side the 1e-2 slack decides (BB_SLACK); half-extents above 2^24 (BB_HUGE);
  centres off screen whose box still reaches in (BB_OFFCENTRE); boxes emptied by the clamp alone (BB_CLAMPED_EMPTY);
  and 1-pixel-wide and 1-pixel-tall viewports.
* SURFEL_*: 2DGS `|d| < 1e-4` and which of sqrt(ex), sqrt(ey), cutoff 0.707106 is the radius.  For a visible
  surfel |d| cannot equal 1e-4f or either of its f32 neighbours: d = (c2 w0^2 + c2 w1^2) - w^2 with w > near = 0.1
  is a difference of two values >= 2^-7, exact and a multiple of 2^-31, while 1e-4f needs 2^-37.  For the w of these
  cases (1 .. 4) the grid is ulp(w^2), about 1e-7: the cases put |d| on grid values below and just above 1e-4.
* EX_* / EY_*: the 2DGS `ex, ey < 1e-4` test with ex (ey) exactly 1e-4f, one ulp above and one below, the other
  extent large.  Reachable where the surfel's mean0 (mean1) is within ~0.01 of 0, where ex's grid is fine enough.
* SIG0_*: Sigma exactly zero, its entries zeros of either sign, seen from general directions: where T Sigma T^t and
  Sigma differ in a zero's sign, the USE_AABB conic's b term (a signed zero) follows it, so an identity shortcut
  taken on a zero entry changes the record.
* KEY_*: key-gen far from the frustum bounds: d2 overflowing to inf (every such key 0xFFFFFFFF - 0x7F800000, ties
  broken by index), clip w across [1e-30, 1e30] (rcp.approx.ftz's window), non-finite positions and finite
  positions whose |x| + |y| + |z| overflows (`keygen_world_pos`'s identity shortcut must not be taken).
* DEPTH_*: the Depth colour range, literal `sorted[1]` / `sorted[N-1]`, with and without culled gaussians, n_vis of
  0, 1 and >= 2, distances chosen so that a wrong entry moves the colours by far more than any tolerance.
* SH_ONEHOT: for each of the 48 coefficients, gaussians whose only non-zero coefficient is that one, seen along the
  axes, on the basis functions' zeros and in general directions.

`colour_bound` is the per-record bound on |CUDA colour - oracle colour| the SH path allows (rsqrt.approx
normalisations, fma accumulation, __powf); see its docstring.
"""
from __future__ import annotations

import dataclasses
import functools
import math

import numpy as np

import bevy_gaussian_splatting_b200 as B

f32 = np.float32
U = 2.0 ** -24                 # unit roundoff of f32
NEAR = 0.1

# geometry name -> (gaussian_mode, aabb)
GEOMETRIES = {"obb3d": (B.GaussianMode.Gaussian3d, False), "aabb3d": (B.GaussianMode.Gaussian3d, True),
              "obb2d": (B.GaussianMode.Gaussian2d, False), "aabb2d": (B.GaussianMode.Gaussian2d, True)}


@dataclasses.dataclass
class Case:
    name: str
    cloud: B.PlanarGaussian3d
    view: object
    model: np.ndarray | None           # row-major 4x4 (None: identity)
    layout: str                        # "f32" | "f16" | "cov"
    settings: dict                     # CloudSettings keywords the case is built for (geometry is added by the test)
    geoms: tuple = tuple(GEOMETRIES)
    tags: dict = dataclasses.field(default_factory=dict)

    @property
    def transform(self):
        return None if self.model is None else B.CloudTransform(self.model)

    def oracle_cloud(self):
        """The planes the oracle reads: what the layout decodes to on the GPU."""
        if self.layout == "f16":
            return self.cloud.rounded_to_f16()
        if self.layout == "cov":
            return self.cloud.precomputed_covariance().rounded_to_f16()
        return self.cloud


class RawCovariance(B.PlanarGaussian3d):
    """A cloud already laid out as Covariance3dOpacity (rotation = c0..c3, scale_opacity = c4, c5, opacity, opacity):
    uploads any record, positive definite or not, through the precomputed-covariance layout."""

    def precomputed_covariance(self):
        return B.PlanarGaussian3d(self.position_visibility, self.spherical_harmonic, self.rotation, self.scale_opacity)


def settings(geom: str, **kw) -> B.CloudSettings:
    gm, aabb = GEOMETRIES[geom]
    return B.CloudSettings(gaussian_mode=gm, aabb=aabb, binning_rounds=False, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# views, models, placement

def axis_view(w=192, h=128):
    """Camera at (0, 0, 5) looking down -z: view-space axes are the world axes, so products with the view matrix
    keep exact zeros (what the sign-of-zero cases need)."""
    return B.perspective_view((0.0, 0.0, 5.0), (0.0, 0.0, 0.0), w, h)


def off_view(w=200, h=136):
    return B.orbit_view(1, 8, w, h)


def model_matrix(kind: str) -> np.ndarray | None:
    """'identity' -> None; 'affine': off-axis, rotated, non-uniformly scaled, translated; 'mirror': the same with a
    negative determinant."""
    if kind == "identity":
        return None
    ax = np.array([0.3, 0.8, -0.5]); ax /= np.linalg.norm(ax)
    a = 0.9
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    R = np.eye(3) + math.sin(a) * K + (1 - math.cos(a)) * K @ K
    S = np.diag([1.3, 0.7, 1.1] if kind == "affine" else [-1.2, 0.9, 1.05])
    m = np.eye(4)
    m[:3, :3] = R @ S
    m[:3, 3] = [0.4, -0.3, 0.6]
    return m.astype(np.float32)


def place(view, ndc_xy, dist, model=None):
    """Cloud-space positions whose world position is at the given ndc (x, y) and distance from the eye (f64 maths,
    rounded to f32: the result lies within a rounding of the target)."""
    ndc_xy = np.asarray(ndc_xy, np.float64).reshape(-1, 2)
    dist = np.broadcast_to(np.asarray(dist, np.float64), (len(ndc_xy),))
    P = view.clip_from_view.astype(np.float64)
    vx = ndc_xy[:, 0] / P[0, 0]
    vy = ndc_xy[:, 1] / P[1, 1]
    d = np.stack([vx, vy, -np.ones_like(vx)], 1)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    pv = d * dist[:, None]
    Vinv = np.linalg.inv(view.view_from_world.astype(np.float64))
    pw = (Vinv[:3, :3] @ pv.T).T + Vinv[:3, 3]
    if model is not None:
        Mi = np.linalg.inv(model.astype(np.float64))
        pw = (Mi[:3, :3] @ pw.T).T + Mi[:3, 3]
    return pw


def cloud_of(pos, rot=None, so=None, sh=None, vis=None, seed=0):
    n = len(pos)
    rng = np.random.default_rng(seed)
    pv = np.ones((n, 4), np.float64)
    pv[:, :3] = pos
    if vis is not None:
        pv[:, 3] = vis
    if rot is None:
        rot = rng.uniform(-1, 1, (n, 4))
    if so is None:
        so = np.concatenate([rng.uniform(0.02, 0.2, (n, 3)), rng.uniform(0.1, 0.9, (n, 1))], 1)
    if sh is None:
        sh = rng.uniform(-1, 1, (n, 48))
    with np.errstate(over="ignore", invalid="ignore"):
        return B.PlanarGaussian3d(pv.astype(f32), np.asarray(sh).astype(f32), np.asarray(rot).astype(f32),
                                  np.asarray(so).astype(f32))


def concat(*clouds):
    return B.PlanarGaussian3d(*(np.concatenate([getattr(c, k) for c in clouds]) for k in
                                ("position_visibility", "spherical_harmonic", "rotation", "scale_opacity")))


def ulp_walk(x, steps):
    """f32 values `steps` ulps from each x (x finite, non-zero and of one sign per row)."""
    b = np.asarray(x, f32).view(np.int32).astype(np.int64)
    return (b[..., None] + np.asarray(steps)[None, :]).astype(np.int32).view(f32)


# ---------------------------------------------------------------------------------------------------------------------
# numpy f32 restatements of the decision quantities (the oracle's operation order, no contraction)

def sigma_f32(rot, so, global_scale=1.0):
    """Sigma = M^T M, M = S R (gaussian_3d.wgsl:49-72, project.cu `sigma3d`) -> (n, 3, 3) f32."""
    q = rot.astype(f32)
    sc = (so[:, :3].astype(f32) * f32(global_scale)).astype(f32)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    one, two = f32(1), f32(2)
    R = np.empty((len(q), 3, 3), f32)
    with np.errstate(all="ignore"):
        R[:, 0, 0] = one - two * (y * y + z * z); R[:, 1, 0] = two * (x * y - r * z); R[:, 2, 0] = two * (x * z + r * y)
        R[:, 0, 1] = two * (x * y + r * z); R[:, 1, 1] = one - two * (x * x + z * z); R[:, 2, 1] = two * (y * z - r * x)
        R[:, 0, 2] = two * (x * z - r * y); R[:, 1, 2] = two * (y * z + r * x); R[:, 2, 2] = one - two * (x * x + y * y)
        M = (sc[:, :, None] * R).astype(f32)
        S = np.empty_like(R)
        for i in range(3):
            for j in range(3):
                S[:, i, j] = (M[:, 0, i] * M[:, 0, j] + M[:, 1, i] * M[:, 1, j]) + M[:, 2, i] * M[:, 2, j]
    return S


def sandwich_f32(A, S):
    """T Sigma T^t with T = A (3x3 f32), the full path of project.cu's `sigma3d`."""
    X = np.empty_like(S)
    TS = np.empty_like(S)
    with np.errstate(all="ignore"):
        for i in range(3):
            for j in range(3):
                X[:, i, j] = (A[i, 0] * S[:, 0, j] + A[i, 1] * S[:, 1, j]) + A[i, 2] * S[:, 2, j]
        for i in range(3):
            for j in range(3):
                TS[:, i, j] = (X[:, i, 0] * A[j, 0] + X[:, i, 1] * A[j, 1]) + X[:, i, 2] * A[j, 2]
    return TS


def cutoff_f32(oracle, opacity):
    """(a, cutoff) of gaussian.wgsl:228-232 in the oracle's f32 arithmetic (a = 9 + 2 ln o, ln = the fixed series)."""
    ln = np.array([oracle.load().orc_ln(float(o)) for o in np.asarray(opacity, f32).ravel()], f32)
    with np.errstate(invalid="ignore"):
        a = (f32(9.0) + f32(2.0) * ln).astype(f32)
        c = np.sqrt(np.where(a > f32(1e-6), a, f32(1e-6))).astype(f32)
    return a, c


def surfel_f32(case_cloud, view, model, cutoff):
    """2DGS homography quantities of gaussian_2d.wgsl:77-132 as project.cu's `surfel_record` evaluates them, in f32:
    -> dict(d, mean0, mean1, ex, ey) (mean / ex / ey are meaningful where |d| >= 1e-4)."""
    q = case_cloud.rotation
    so = case_cloud.scale_opacity
    A = np.eye(3, dtype=f32) if model is None else model[:3, :3].astype(f32)
    t = np.zeros(3, f32) if model is None else model[:3, 3].astype(f32)
    R = sigma_rows(q)
    sc = so[:, :3].astype(f32)
    CW = view.clip_from_world.astype(f32)
    W, H = f32(view.width), f32(view.height)
    P = view.clip_from_view.astype(f32)
    p = case_cloud.position_visibility[:, :3].astype(f32)
    with np.errstate(all="ignore"):
        pw = [((A[r, 0] * p[:, 0] + A[r, 1] * p[:, 1]) + A[r, 2] * p[:, 2]) + t[r] for r in range(3)]
        G = []                                                      # G[j][r]: clip row r of column j
        for j in range(2):
            rc = [R[:, j, k] * sc[:, j] for k in range(3)]
            Lj = [(A[i, 0] * rc[0] + A[i, 1] * rc[1]) + A[i, 2] * rc[2] for i in range(3)]
            G.append([(CW[r, 0] * Lj[0] + CW[r, 1] * Lj[1]) + CW[r, 2] * Lj[2] for r in range(4)])
        G.append([((CW[r, 0] * pw[0] + CW[r, 1] * pw[1]) + CW[r, 2] * pw[2]) + CW[r, 3] for r in range(4)])
        fxk, fyk = (P[0, 0] * W) / f32(2), (P[1, 1] * H) / f32(2)
        cxk, cyk = (W - f32(1)) / f32(2), (H - f32(1)) / f32(2)
        T0 = [fxk * G[j][0] + cxk * G[j][3] for j in range(3)]
        T1 = [fyk * G[j][1] + cyk * G[j][3] for j in range(3)]
        T2 = [G[j][3] for j in range(3)]
        c2 = f32(cutoff) * f32(cutoff)
        test = [c2, c2, f32(-1.0)]
        dot3 = lambda u, v: (u[0] * v[0] + u[1] * v[1]) + u[2] * v[2]
        d = dot3([test[k] * T2[k] for k in range(3)], T2)
        inv = f32(1) / d
        f = [inv * test[k] for k in range(3)]
        mean0 = dot3(f, [T0[k] * T2[k] for k in range(3)])
        mean1 = dot3(f, [T1[k] * T2[k] for k in range(3)])
        ex = mean0 * mean0 - dot3([f[k] * T0[k] for k in range(3)], T0)
        ey = mean1 * mean1 - dot3([f[k] * T1[k] for k in range(3)], T1)
    return {k: np.asarray(v, f32) for k, v in dict(d=d, mean0=mean0, mean1=mean1, ex=ex, ey=ey).items()}


def surfel_d_f32(case_cloud, view, model, cutoff):
    return surfel_f32(case_cloud, view, model, cutoff)["d"]


def sigma_rows(q):
    """Rotation matrix rows (helpers.wgsl:137-158, (row, col)) in f32."""
    q = q.astype(f32)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    one, two = f32(1), f32(2)
    R = np.empty((len(q), 3, 3), f32)
    with np.errstate(all="ignore"):
        R[:, 0, 0] = one - two * (y * y + z * z); R[:, 1, 0] = two * (x * y - r * z); R[:, 2, 0] = two * (x * z + r * y)
        R[:, 0, 1] = two * (x * y + r * z); R[:, 1, 1] = one - two * (x * x + z * z); R[:, 2, 1] = two * (y * z - r * x)
        R[:, 0, 2] = two * (x * z - r * y); R[:, 1, 2] = two * (y * z + r * x); R[:, 2, 2] = one - two * (x * x + y * y)
    return R


def bbox_args(cx, cy, hx, hy):
    """The four ceil / floor arguments of make_bbox (project.cu:49-63) in f32: (x0, x1, y0, y1) arguments."""
    cx, cy, hx, hy = (np.asarray(v, f32) for v in (cx, cy, hx, hy))
    with np.errstate(all="ignore"):
        sx = hx * f32(1e-3) + f32(1e-2)
        sy = hy * f32(1e-3) + f32(1e-2)
        return ((cx - hx) - (f32(0.5) + sx), (cx + hx) - (f32(0.5) - sx), (cy - hy) - (f32(0.5) + sy),
                (cy + hy) - (f32(0.5) - sy))


def oracle_records(oracle, case: Case, geom: str, **kw):
    """The oracle's record of every gaussian of the case (visible or not), in cloud order."""
    s = settings(geom, **{**case.settings, **kw})
    s_abi = s.to_abi()
    s_abi.reserved = 1 if case.layout == "cov" else 0
    u = B.GaussianSplattingPlugin.cloud_uniform(s, case.transform)
    oc = case.oracle_cloud()
    return oracle.project(oc, case.view.to_abi(), u, s_abi, np.arange(len(oc), dtype=np.uint32))


def drawn_of(rec):
    return rec["xlo"] <= rec["xhi"]


# ---------------------------------------------------------------------------------------------------------------------
# the cases

def draw_mode_case(seed=0):
    """The visibility lane around 0.5 and at its special values, 64 gaussians per value, scattered over the frame."""
    half = f32(0.5)
    vals = np.array([half, np.nextafter(half, f32(0)), np.nextafter(half, f32(1)), 0.0, -0.0, -1.0, 1.0, 0.49999,
                     np.nan, np.inf, -np.inf, 2.0], f32)
    rng = np.random.default_rng(100 + seed)
    view = off_view()
    k = 64
    w = np.repeat(vals, k)
    pos = place(view, rng.uniform(-0.9, 0.9, (len(w), 2)), rng.uniform(2.0, 9.0, len(w)))
    c = cloud_of(pos, vis=w, seed=seed)
    c.position_visibility[:, 3] = w            # (-0 and NaN survive the f32 cast above, but keep them exact)
    wb = w.view(np.uint32)
    tags = {"DRAW_HALF": w == half, "DRAW_BELOW": w == np.nextafter(half, f32(0)), "DRAW_ABOVE": w == np.nextafter(half, f32(1)),
            "DRAW_NEGZERO": wb == 0x80000000, "DRAW_NEG": w < 0, "DRAW_NAN": np.isnan(w), "DRAW_INF": np.isinf(w)}
    return [Case(f"draw_{m.name}", c, view, None, "f32", dict(draw_mode=m), tags=tags)
            for m in (B.DrawMode.Selected, B.DrawMode.HighlightSelected)]


def cutoff_case(oracle, seed=0):
    """f32 opacities on both sides of the adaptive-cutoff clamp, and the special opacities."""
    o0 = f32(math.exp(-4.5))
    cand = ulp_walk(o0, np.arange(-40, 41))[0]
    a, _ = cutoff_f32(oracle, cand)
    last_clamped = cand[a <= f32(1e-6)].max()
    first_kept = cand[a > f32(1e-6)].min()
    specials = np.array([0.0, -0.0, -0.25, 1e-40, np.nan, np.inf, 1.0, 1.5, 7.0, 0.8], f32)
    ops = np.concatenate([cand, specials, [last_clamped] * 8, [first_kept] * 8]).astype(f32)
    rng = np.random.default_rng(200 + seed)
    view = off_view()
    n = len(ops)
    pos = place(view, rng.uniform(-0.9, 0.9, (n, 2)), rng.uniform(2.0, 6.0, n))
    so = np.concatenate([rng.uniform(0.03, 0.2, (n, 3)), ops[:, None]], 1)
    c = cloud_of(pos, so=so, seed=seed)
    c.scale_opacity[:, 3] = ops
    a, _ = cutoff_f32(oracle, ops)
    with np.errstate(invalid="ignore"):
        tags = {"CUT_LAST_CLAMPED": ops == last_clamped, "CUT_FIRST_KEPT": ops == first_kept,
                "CUT_A_ZERO": a == 0, "CUT_CLAMPED": ~(a > f32(1e-6)), "CUT_KEPT": a > f32(1e-6),
                "O_ZERO": ops == 0, "O_NEG": ops < 0, "O_NAN": np.isnan(ops), "O_GT1": ops > 1,
                "O_SUBNORMAL": (ops != 0) & (np.abs(ops) < np.finfo(f32).tiny)}
    return [Case("cutoff", c, view, None, "f32", dict(opacity_adaptive_radius=True), tags=tags)]


def _signed_zero_quats():
    """Quaternions with exact zeros of both signs: axis-aligned frames (and 90-degree turns) whose R has +-0 entries."""
    z, nz, h = 0.0, -0.0, math.sqrt(0.5)
    out = [(1, z, z, z), (1, nz, z, z), (1, z, nz, z), (1, z, z, nz), (-1, nz, nz, nz), (nz, 1, z, z), (z, nz, 1, z),
           (z, z, nz, 1), (h, h, z, z), (h, z, nz, h), (h, nz, z, h), (-h, z, h, nz)]
    return np.array(out, f32)


def _negzero_sigmas():
    """(quaternion, scale) pairs over {+-1, +-0} quaternions and signed scales whose Sigma has a -0 entry (found by
    exhaustive search in the f32 restatement)."""
    vals = np.array([1.0, -1.0, 0.0, -0.0], f32)
    q = np.array(np.meshgrid(vals, vals, vals, vals, indexing="ij"), f32).reshape(4, -1).T
    sc = np.array(np.meshgrid([0.05, -0.05], [0.12, -0.12], [0.02, -0.02], indexing="ij"), f32).reshape(3, -1).T
    Q = np.repeat(q, len(sc), 0)
    S3 = np.tile(sc, (len(q), 1))
    so = np.concatenate([S3, np.ones((len(S3), 1), f32)], 1)
    e = sigma_f32(Q, so)[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
    neg = np.any(e.view(np.uint32) == 0x80000000, 1) & np.isfinite(e).all(1)
    idx = np.flatnonzero(neg)[::max(1, int(neg.sum()) // 24)]
    # and rows with Sigma01 = -0, Sigma00 != Sigma11 (each twice: once on the axis view's axis, once off it)
    s01 = np.flatnonzero((e[:, 1].view(np.uint32) == 0x80000000) & (e[:, 0] != e[:, 3]) & np.isfinite(e).all(1))
    s01 = np.repeat(s01[::max(1, len(s01) // 12)], 2)
    idx = np.concatenate([idx, s01])
    return Q[idx], S3[idx]


def sigma_case(seed=0):
    """Identity model, axis view: Sigma with zero, -0, subnormal, infinite and NaN entries (the identity shortcut
    must not be taken) next to ordinary ones (it is).  Splats sit on the view axis and off it."""
    rng = np.random.default_rng(300 + seed)
    view = axis_view()
    qs = _signed_zero_quats()
    scales = np.array([[0.05, 0.12, 0.02], [-0.05, 0.12, 0.02], [0.07, -0.07, 0.0], [0.0, 0.0, 0.0], [-0.0, 0.1, 0.03],
                       [1e-23, 0.08, 0.04], [2e-20, 3e-21, 0.05], [1e20, 0.05, 0.05], [0.1, np.inf, 0.1],
                       [0.1, np.nan, 0.1], [0.09, 0.09, 0.09], [0.05, 0.05, 1e-3]], f32)
    rot, so = [], []
    for q in qs:
        for s in scales:
            rot.append(q); so.append(s)
    nq, ns = _negzero_sigmas()
    rot = np.concatenate([np.array(rot, f32), nq]); so3 = np.concatenate([np.array(so, f32), ns])
    # and general splats (shortcut taken), plus NaN / inf quaternions
    ng = 120
    rot = np.concatenate([rot, rng.uniform(-1, 1, (ng, 4)).astype(f32),
                          np.array([[np.nan, 0, 0, 1], [1, np.inf, 0, 0], [1e20, 0, 0, 0], [1e-22, 0, 0, 0]], f32)])
    so3 = np.concatenate([so3, rng.uniform(0.02, 0.2, (ng, 3)).astype(f32), np.full((4, 3), 0.06, f32)])
    n = len(rot)
    # half on the axis (x = y = 0: exact zeros in the Jacobian), half off it
    ndc = np.where((np.arange(n) % 2 == 0)[:, None], 0.0, rng.uniform(-0.8, 0.8, (n, 2)))
    pos = place(view, ndc, rng.uniform(2.0, 6.0, n))
    pos[np.arange(n) % 2 == 0, :2] = 0.0
    so = np.concatenate([so3, rng.uniform(0.3, 0.9, (n, 1))], 1)
    c = cloud_of(pos, rot=rot, so=so, seed=seed)
    c.rotation[:] = rot
    c.scale_opacity[:, :3] = so3
    S = sigma_f32(c.rotation, c.scale_opacity)
    e = S[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
    with np.errstate(invalid="ignore"):
        ae = np.abs(e)
        shortcut = np.all(ae > 0, 1) & np.all(np.isfinite(e), 1)
        full = sandwich_f32(np.eye(3, dtype=f32), S)[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
        tags = {"SIG_SHORTCUT": shortcut, "SIG_ZERO": np.any(e == 0, 1),
                "SIG_NEGZERO": np.any(e.view(np.uint32) == 0x80000000, 1),
                "SIG_SUBNORMAL": np.any((ae > 0) & (ae < np.finfo(f32).tiny), 1), "SIG_INF": np.any(np.isinf(e), 1),
                "SIG_NAN": np.any(np.isnan(e), 1),
                "SIG_SIGNZERO": ~shortcut & np.all(np.isfinite(e), 1) & np.any(full.view(np.uint32) != e.view(np.uint32), 1)}
    return [Case("sigma", c, view, None, "f32", dict(opacity_adaptive_radius=False), tags=tags)]


def obb_case(oracle, model_kind="identity", seed=0):
    """Axis-aligned splats on and off the axis view's axis (b = +-0 with a != c, and a = c: the NaN eigenvector),
    needles and near-plane splats (the minor axis rounds to 0 or NaN), degenerate and overflowing conics."""
    rng = np.random.default_rng(400 + seed)
    view = axis_view()
    model = model_matrix(model_kind)
    one = np.array([1, 0, 0, 0], f32)
    rows = []
    for s in ([0.1, 0.1, 0.1], [0.1, 0.05, 0.02], [0.03, 0.2, 0.1], [0.07, 0.07, 0.3], [0.0, 0.0, 0.0], [0.2, 0.0, 0.0],
              [3.0, 1e-4, 1e-4], [30.0, 1e-6, 0.0], [1e-5, 40.0, 1e-5], [1e15, 1e15, 1e15], [1e18, 0.1, 0.1],
              [5e17, 5e17, 0.0]):
        for on_axis in (True, False):
            for q in (one, np.array([0.7, 0.0, 0.0, 0.7], f32), np.array([0.9, 0.3, -0.2, 0.1], f32)):
                rows.append((s, on_axis, q))
    n = len(rows)
    so = np.array([list(r[0]) + [0.7] for r in rows], f32)
    rot = np.array([r[2] for r in rows], f32)
    on = np.array([r[1] for r in rows])
    ndc = np.where(on[:, None], 0.0, rng.uniform(-0.7, 0.7, (n, 2)))
    pos = place(view, ndc, rng.uniform(0.3, 6.0, n), model)
    if model is None:
        pos[on, :2] = 0.0
    c = cloud_of(pos, rot=rot, so=so, seed=seed)
    c.rotation[:] = rot
    c.scale_opacity[:] = so
    case = Case(f"obb_{model_kind}", c, view, model, "f32", dict(opacity_adaptive_radius=False))
    obb = oracle_records(oracle, case, "obb3d")
    aab = oracle_records(oracle, case, "aabb3d")
    with np.errstate(invalid="ignore"):
        conic = np.stack([aab["extra"][:, 0], aab["extra"][:, 1], aab["extra"][:, 2]], 1)
        case.tags = {
            "B0_ANEC": (conic[:, 1] == 0) & (conic[:, 0] != conic[:, 2]) & np.isfinite(conic).all(1),
            "EV_NAN": np.isnan(obb["ux"]) & ~drawn_of(obb) & np.isfinite(conic).all(1),
            "MINOR_NONFINITE": drawn_of(obb) & ~(np.isfinite(obb["vx"]) & np.isfinite(obb["vy"])),
            "DET_ZERO": drawn_of(aab) & np.isinf(conic).any(1),
            "DET_NAN": drawn_of(aab) & np.isnan(conic).any(1),
        }
    return case


def bbox_case(oracle, seed=0):
    """USE_AABB splats whose bbox edges are walked onto integers: the x position moves one f32 ulp at a time and the
    oracle's centre and quad half-side are read back, until an edge's ceil / floor argument is an integer, one ulp
    above or below one, or within the slack's 1e-3 px on the side it decides.  Plus huge half-extents, off-screen
    centres whose box reaches in, boxes emptied by the clamp."""
    rng = np.random.default_rng(500 + seed)
    view = off_view(160, 96)
    n0 = 48
    ndc = rng.uniform(-0.85, 0.85, (n0, 2))
    dist = rng.uniform(2.0, 6.0, n0)
    base = place(view, ndc, dist)
    so = np.array([0.03, 0.05, 0.04, 0.8], f32)
    rot = np.array([0.8, 0.1, -0.3, 0.2], f32)

    def x0_args(steps):
        cand = ulp_walk(base[:, 0].astype(f32), steps)                # (n0, S)
        pos = np.repeat(base, cand.shape[1], 0)
        pos[:, 0] = cand.ravel()
        probe = Case("probe", cloud_of(pos, rot=np.tile(rot, (len(pos), 1)), so=np.tile(so, (len(pos), 1)), seed=seed),
                     view, None, "f32", dict(opacity_adaptive_radius=False))
        rec = oracle_records(oracle, probe, "aabb3d")
        h = (f32(0.5) * rec["extra"][:, 3]).astype(f32)
        x0a, x1a, _, _ = bbox_args(rec["cx"], rec["cy"], h, h)
        return pos, x0a.reshape(n0, -1), x1a.reshape(n0, -1)

    # coarse: the x0 argument is linear in the ulp step over this range; aim at the nearest integer above it
    _, c0, _ = x0_args(np.array([0, 4096]))
    slope = (c0[:, 1].astype(np.float64) - c0[:, 0]) / 4096.0
    aim = np.round((np.ceil(c0[:, 0].astype(np.float64)) - c0[:, 0]) / slope).astype(np.int64)
    base[:, 0] = (base[:, 0].astype(f32).view(np.int32).astype(np.int64) + aim).astype(np.int32).view(f32)
    steps = np.arange(-400, 401)
    pos, x0a, x1a = x0_args(steps)
    k = len(steps)
    pick = []
    for i in range(n0):
        a0 = x0a[i]
        fr = a0 - np.floor(a0)
        du = (a0.astype(np.float64) - np.round(a0)) / np.spacing(np.abs(a0))
        for want in ((du == 0), (du >= 1) & (du <= 4), (du <= -1) & (du >= -4)):      # on, just above, just below
            hit = np.flatnonzero(want)
            if len(hit):
                pick.append(i * k + hit[len(hit) // 2])
        sl_lo = np.flatnonzero((fr > 0) & (fr <= 1e-3))
        if len(sl_lo):
            pick.append(i * k + sl_lo[0])
        a1 = x1a[i]
        fr1 = np.ceil(a1) - a1
        sl_hi = np.flatnonzero((fr1 > 0) & (fr1 <= 1e-3))
        if len(sl_hi):
            pick.append(i * k + sl_hi[0])
    pick = np.unique(np.array(pick, np.int64))
    pos_k = pos[pick]
    # huge half-extents (> 2^24 px), off-screen centres that still reach in, boxes emptied by the clamp
    m = 24
    big = place(view, rng.uniform(-0.5, 0.5, (m, 2)), rng.uniform(0.3, 1.0, m))
    off = place(view, np.stack([rng.choice([-1.09, 1.09, -1.05, 1.05], m), rng.uniform(-0.8, 0.8, m)], 1), rng.uniform(2, 5, m))
    clamp = place(view, np.stack([rng.choice([-1.06, 1.06, -1.09, 1.09], m), rng.uniform(-0.8, 0.8, m)], 1), rng.uniform(2, 5, m))
    allpos = np.concatenate([pos_k, big, off, clamp])
    nk = len(pos_k)
    so_all = np.tile(so, (len(allpos), 1))
    so_all[nk:nk + m, :3] = rng.uniform(1e5, 1e7, (m, 3))
    so_all[nk + m:nk + 2 * m, :3] = rng.uniform(0.3, 0.8, (m, 3))
    so_all[nk + 2 * m:, :3] = rng.uniform(1e-3, 4e-3, (m, 3))
    c = cloud_of(allpos, rot=np.tile(rot, (len(allpos), 1)), so=so_all, seed=seed)
    case = Case("bbox", c, view, None, "f32", dict(opacity_adaptive_radius=False))
    rec = oracle_records(oracle, case, "aabb3d")
    h = (f32(0.5) * rec["extra"][:, 3]).astype(f32)
    args = bbox_args(rec["cx"], rec["cy"], h, h)
    with np.errstate(invalid="ignore"):
        ulp = lambda a: np.spacing(np.abs(a)).astype(f32)
        on = np.zeros(len(c), bool); up = np.zeros(len(c), bool); down = np.zeros(len(c), bool); slack = np.zeros(len(c), bool)
        small = np.ones(len(c), bool)
        small[-3 * m:] = False                  # (huge boxes' arguments are integers for want of fraction bits)
        for a in args:
            du = (a.astype(np.float64) - np.round(a)) / ulp(a)
            on |= small & (du == 0)
            up |= small & (du >= 1) & (du <= 4)
            down |= small & (du <= -1) & (du >= -4)
        slack |= ((args[0] - np.floor(args[0])) > 0) & ((args[0] - np.floor(args[0])) <= 1e-3)
        slack |= ((np.ceil(args[1]) - args[1]) > 0) & ((np.ceil(args[1]) - args[1]) <= 1e-3)
        vis = ~np.isnan(rec["cx"]) & (rec["extra"][:, 3] > 0)
        x0, x1, y0, y1 = np.ceil(args[0]), np.floor(args[1]), np.ceil(args[2]), np.floor(args[3])
        pre = (x0 <= x1) & (y0 <= y1)
        W, H = view.width, view.height
        post = (np.maximum(x0, 0) <= np.minimum(x1, W - 1)) & (np.maximum(y0, 0) <= np.minimum(y1, H - 1))
        case.tags = {"BB_ON": on & vis, "BB_UP": up & vis, "BB_DOWN": down & vis, "BB_SLACK": slack & vis,
                     "BB_HUGE": vis & (h > 2.0 ** 24) & drawn_of(rec),
                     "BB_OFFCENTRE": drawn_of(rec) & ((rec["cx"] < 0) | (rec["cx"] > W)),
                     "BB_CLAMPED_EMPTY": vis & pre & ~post}
    return case


def thin_viewport_cases(seed=0):
    """1-pixel-wide and 1-pixel-tall frames."""
    out = []
    for w, h in ((1, 48), (48, 1)):
        view = B.perspective_view((0.3, 0.2, 5.0), (0.0, 0.0, 0.0), w, h)
        rng = np.random.default_rng(600 + seed + w)
        n = 400
        pos = place(view, rng.uniform(-1.05, 1.05, (n, 2)), rng.uniform(2.0, 8.0, n))
        c = cloud_of(pos, seed=seed)
        c.scale_opacity[:, :3] *= f32(0.3)
        out.append(Case(f"viewport_{w}x{h}", c, view, None, "f32", {}, tags={"VIEWPORT_THIN": np.ones(n, bool)}))
    return out


def surfel_case(seed=0):
    """Surfels turned edge-on (d -> 0): for each of a few positions, the surfel's normal is walked through the view
    direction so that |d| takes the f32 grid values on both sides of 1e-4; tiny surfels whose radius is the cutoff
    0.707106 floor; surfels where sqrt(ex) or sqrt(ey) wins; extents walked down to 1e-4."""
    rng = np.random.default_rng(700 + seed)
    view = off_view()
    model = model_matrix("affine")
    n0 = 24
    ndc = rng.uniform(-0.7, 0.7, (n0, 2))
    dist = rng.uniform(1.0, 4.0, n0)
    pos = place(view, ndc, dist, model)
    # quaternion (cos t, sin t * axis): walk t so that the surfel plane contains the ray
    ts = np.linspace(-np.pi, np.pi, 721)
    ax = rng.normal(size=(n0, 3)); ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    cand_q = np.concatenate([np.cos(ts)[None, :, None] * np.ones((n0, 1, 1)),
                             np.sin(ts)[None, :, None] * ax[:, None, :]], 2).reshape(-1, 4)
    P = np.repeat(pos, len(ts), 0)
    # axes of about w / 3 (the model scales by 0.7 .. 1.3): 9 (w0^2 + w1^2) - w^2 changes sign as the surfel turns
    so_i = np.stack([0.45 * dist, 0.4 * dist, np.zeros(n0), np.full(n0, 0.8)], 1).astype(f32)
    so = np.repeat(so_i, len(ts), 0)
    probe = cloud_of(P, rot=cand_q, so=so, seed=seed)
    d = surfel_d_f32(probe, view, model, 3.0).reshape(n0, len(ts))
    picks = []
    thr = f32(1e-4)
    for i in range(n0):
        # bracket each sign change of d, then refine t in f64 and walk the f32 quaternion component
        s = np.flatnonzero(np.sign(d[i, :-1]) != np.sign(d[i, 1:]))
        for j in s[:2]:
            lo, hi = ts[j], ts[j + 1]
            for _ in range(60):
                mid = 0.5 * (lo + hi)
                qm = np.concatenate([[math.cos(mid)], math.sin(mid) * ax[i]])[None]
                dm = surfel_d_f32(cloud_of(pos[i:i + 1], rot=qm, so=so_i[i:i + 1]), view, model, 3.0)[0]
                if np.sign(dm) == np.sign(d[i, j]):
                    lo = mid
                else:
                    hi = mid
            q0 = np.concatenate([[math.cos(lo)], math.sin(lo) * ax[i]]).astype(f32)
            walk = ulp_walk(q0[0:1], np.arange(-4000, 4001, 7))[0]
            qq = np.tile(q0, (len(walk), 1)); qq[:, 0] = walk
            dd = surfel_d_f32(cloud_of(np.repeat(pos[i:i + 1], len(walk), 0), rot=qq, so=np.repeat(so_i[i:i + 1], len(walk), 0)),
                              view, model, 3.0)
            ad = np.abs(dd)
            below = np.flatnonzero(ad < thr)
            above = np.flatnonzero(ad >= thr)
            if len(below) and len(above):
                b_ = below[np.argmax(ad[below])]
                a_ = above[np.argmin(ad[above])]
                picks += [(i, qq[b_]), (i, qq[a_])]
    pos_k = np.array([pos[i] for i, _ in picks]).reshape(-1, 3)
    rot_k = np.array([q for _, q in picks], f32).reshape(-1, 4)
    so_k = np.array([so_i[i] for i, _ in picks], f32).reshape(-1, 4)
    # radius classes: tiny surfels (cutoff floor), elongated (sqrt ex or sqrt ey wins), extents walked towards 1e-4
    m = 96
    pos_r = place(view, rng.uniform(-0.8, 0.8, (m, 2)), rng.uniform(2.0, 8.0, m), model)
    sc = np.concatenate([rng.uniform(1e-4, 2e-3, (m // 3, 2)), np.stack([rng.uniform(0.05, 0.3, m // 3), rng.uniform(1e-4, 1e-3, m // 3)], 1),
                         np.stack([rng.uniform(1e-4, 1e-3, m // 3), rng.uniform(0.05, 0.3, m // 3)], 1)])
    rot_r = rng.uniform(-1, 1, (m, 4)).astype(f32)
    allpos = np.concatenate([pos_k, pos_r])
    rot = np.concatenate([rot_k, rot_r]).astype(f32)
    so_all = np.tile(np.array([0.05, 0.08, 0.0, 0.8], f32), (len(allpos), 1))
    so_all[:len(pos_k)] = so_k
    so_all[len(pos_k):, :2] = sc
    so_all[len(pos_k):, 2] = 0.01
    c = cloud_of(allpos, rot=rot, so=so_all, seed=seed)
    c.rotation[:] = rot
    d = surfel_d_f32(c, view, model, 3.0)
    ad = np.abs(d)
    case = Case("surfel", c, view, model, "f32", dict(opacity_adaptive_radius=False), geoms=("obb2d", "aabb2d"))
    g = np.float32
    case.tags = {"SURFEL_D_BELOW": ad < thr, "SURFEL_D_ABOVE_NEAR": (ad >= thr) & (ad < g(1.001e-4))}
    return case


def surfel_extent_case(seed=0):
    """Surfels whose ex (or ey) is walked onto 1e-4f and its two f32 neighbours.  ex = mean0^2 - (...) is on a fine
    enough f32 grid only where mean0 is near 0: the surfels sit where mean0 (or mean1) is 0.002 .. 0.012, face the
    axis view's camera, are ~0.01 units wide along the walked axis and long along the other; the walked scale moves one f32 ulp at a time and each candidate is
    evaluated with `surfel_f32` (bit-identical to the oracle's record)."""
    rng = np.random.default_rng(750 + seed)
    view = axis_view()
    W, H = view.width, view.height
    thr = f32(1e-4)
    pos_out, so_out = [], []
    for axis in (0, 1):                     # 0: walk the x scale (ex), 1: the y scale (ey)
        n0 = 24
        px = rng.uniform(0.002, 0.012, n0)                 # pixel coordinate of the centre on the walked axis
        other = rng.uniform(0.3, 0.7, n0)
        # mean = (p_axis * size / 2) ndc + (size - 1) / 2 (the intrinsics of helpers.wgsl:122-135 applied to clip
        # space, so the projection's scale enters twice): solve for the ndc whose mean is px
        P = view.clip_from_view.astype(np.float64)
        ndc = np.empty((n0, 2))
        ndc[:, axis] = (px - (size := (W, H)[axis]) / 2.0 + 0.5) / (P[axis, axis] * size / 2.0)
        ndc[:, 1 - axis] = other - 0.5
        dist = rng.uniform(2.0, 4.0, n0)
        pos = place(view, ndc, dist)
        so = np.zeros((n0, 4), np.float64)
        so[:, 3] = 0.8
        so[:, 1 - axis] = 0.05 * dist / 3.0                 # ~10 px along the other axis
        so[:, axis] = 6e-5 * dist / 3.0                     # ~0.01 px along the walked one
        so[:, 2] = 1e-3
        rot = np.tile(np.array([1.0, 0.0, 0.0, 0.0]), (n0, 1))
        key = "ex" if axis == 0 else "ey"
        for _ in range(3):                                  # fit: the extent scales with the square of the scale
            e = surfel_f32(cloud_of(pos, rot=rot, so=so), view, None, 3.0)[key].astype(np.float64)
            so[:, axis] *= np.sqrt(np.where(e > 0, 1e-4 / e, 1.0))
        steps = np.arange(-256, 257)
        cand = ulp_walk(so[:, axis].astype(f32), steps)    # (n0, S)
        P = np.repeat(pos, len(steps), 0)
        SO = np.repeat(so, len(steps), 0)
        SO[:, axis] = cand.ravel()
        e = surfel_f32(cloud_of(P, rot=np.repeat(rot, len(steps), 0), so=SO), view, None, 3.0)[key].reshape(n0, -1)
        for i in range(n0):
            du = ulps_between(e[i], thr)
            for want in (0, 1, -1):
                hit = np.flatnonzero(du == want)
                if len(hit):
                    pos_out.append(pos[i]); so_out.append(SO[i * len(steps) + hit[0]])
    pos = np.array(pos_out).reshape(-1, 3)
    so = np.array(so_out, f32).reshape(-1, 4)
    c = cloud_of(pos, rot=np.tile(np.array([1.0, 0.0, 0.0, 0.0]), (len(pos), 1)), so=so, seed=seed)
    c.scale_opacity[:] = so
    q = surfel_f32(c, view, None, 3.0)
    dx, dy = ulps_between(q["ex"], thr), ulps_between(q["ey"], thr)
    big_y, big_x = q["ey"] > f32(1e-3), q["ex"] > f32(1e-3)
    case = Case("surfel_extent", c, view, None, "f32", dict(opacity_adaptive_radius=False), geoms=("obb2d", "aabb2d"))
    case.tags = {"EX_ON": (dx == 0) & big_y, "EX_ABOVE": (dx == 1) & big_y, "EX_BELOW": (dx == -1) & big_y,
                 "EY_ON": (dy == 0) & big_x, "EY_ABOVE": (dy == 1) & big_x, "EY_BELOW": (dy == -1) & big_x}
    return case


def ulps_between(q, thr):
    """Signed distance of f32 q from f32 thr in ulps (positive: q above thr; both positive or zero)."""
    return np.asarray(q, f32).view(np.int32).astype(np.int64) - np.asarray(thr, f32).view(np.int32).astype(np.int64)


def sigma_zero_cases(seed=0):
    """Identity model, Sigma exactly zero (zero scales with +-0 signs and quaternions of +-1 / +-0 components), seen
    from general directions: every Sigma entry is a zero whose sign depends on the rotation and the scale signs, and
    T Sigma T^t turns some -0 into +0.  The USE_AABB conic's b term is then a signed zero fed by those signs; where
    it differs, the identity shortcut taken on a zero Sigma would change the record (tag SIG0_SHORTCUT_CHANGES,
    counted with the oracle by feeding Sigma itself through the covariance path)."""
    vals = np.array([1.0, -1.0, 0.0, -0.0], f32)
    import itertools
    Q = np.array(list(itertools.product(vals, repeat=4)), f32)
    Sc = np.array(list(itertools.product([0.0, -0.0], repeat=3)), f32)
    Q = np.repeat(Q, len(Sc), 0)
    Sc = np.tile(Sc, (len(vals) ** 4, 1))
    so = np.concatenate([Sc, np.full((len(Sc), 1), 0.8, f32)], 1)
    e = sigma_f32(Q, so)[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
    keep = np.unique(e.view(np.uint32), axis=0, return_index=True)[1]    # one (rotation, scale) per sign pattern
    Q, so = Q[keep], so[keep]
    rng = np.random.default_rng(1400 + seed)
    out = []
    for v in range(10):
        eye = rng.normal(size=3)
        eye = eye / np.linalg.norm(eye) * 5.0
        view = B.perspective_view(tuple(eye), (0.0, 0.0, 0.0), 96, 64)
        k = 6
        pos = np.repeat(place(view, rng.uniform(-0.6, 0.6, (k, 2)), rng.uniform(2.0, 6.0, k)), len(Q), 0)
        c = cloud_of(pos, rot=np.tile(Q, (k, 1)), so=np.tile(so, (k, 1)), seed=seed)
        c.rotation[:] = np.tile(Q, (k, 1))
        c.scale_opacity[:] = np.tile(so, (k, 1))
        out.append(Case(f"sigma_zero_{v}", c, view, None, "f32", dict(opacity_adaptive_radius=False),
                        geoms=("obb3d", "aabb3d")))
    return out


def shortcut_changes(oracle, case):
    """Mask of the gaussians whose USE_AABB or OBB record changes when Sigma itself (the identity shortcut's value)
    replaces T Sigma T^t: the covariance path fed with Sigma, against the full path."""
    S = sigma_f32(case.cloud.rotation, case.cloud.scale_opacity)
    e = S[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
    so = case.cloud.scale_opacity
    raw = RawCovariance(case.cloud.position_visibility, case.cloud.spherical_harmonic, e[:, :4],
                        np.concatenate([e[:, 4:], so[:, 3:], so[:, 3:]], 1))
    differ = np.zeros(len(raw), bool)
    for geom in ("obb3d", "aabb3d"):
        full = oracle_records(oracle, case, geom)
        s = settings(geom, **case.settings).to_abi()
        s.reserved = 1
        u = B.GaussianSplattingPlugin.cloud_uniform(settings(geom, **case.settings))
        short = oracle.project(raw, case.view.to_abi(), u, s, np.arange(len(raw), dtype=np.uint32))
        d = np.zeros(len(raw), bool)
        for k in ("cx", "cy", "ux", "uy", "vx", "vy"):
            d |= ~bits_agree(full[k], short[k])
        for j in range(4):
            d |= ~bits_agree(full["extra"][:, j], short["extra"][:, j])
        differ |= d & drawn_of(full)
    return differ


def surfel_radius_tags(oracle, case):
    """Which argument of max(sqrt ex, sqrt ey, cutoff 0.707106) is the radius, read from the oracle's 2DGS record."""
    rec = oracle_records(oracle, case, "aabb2d")
    Rq = rec["extra"][:, 3]
    floor = f32(3.0) * f32(0.707106)
    dr = drawn_of(rec)
    return {"SURFEL_FLOOR": dr & (Rq == floor), "SURFEL_EXTENT": dr & (Rq > floor),
            "SURFEL_REJECTED": ~dr & ~np.isnan(rec["cx"])}


def keygen_far_case(seed=0):
    """Key-gen away from the frustum bounds on an axis view: d2 overflowing (ties by index), clip w across
    [1e-30, 1e30], non-finite positions, finite positions whose |x| + |y| + |z| overflows."""
    rng = np.random.default_rng(800 + seed)
    view = axis_view()
    pts = []
    for dist in (1e18, 1.8e19, 2e19, 1e25, 9e29, 1e30, 1.1e30, 1e31, 1e36, 3.3e38):
        for _ in range(6):
            nd = rng.uniform(-0.8, 0.8, 2)
            pts.append(place(view, nd[None], dist)[0])
    pts = np.array(pts)
    over = np.array([[2e37, 0.0, -3.39e38], [-3e37, 1e37, -3.38e38], [0.0, 0.0, -3.4e38], [1e38, 1e38, -3e38]])
    nonf = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [np.inf, np.inf, -np.inf], [0, 0, np.nan]])
    near = place(view, rng.uniform(-0.8, 0.8, (40, 2)), rng.uniform(0.2, 8.0, 40))
    allp = np.concatenate([near, pts, over, nonf])
    with np.errstate(all="ignore"):
        p32 = allp.astype(f32)
        c = cloud_of(p32, seed=seed)
        x, y, z = p32[:, 0], p32[:, 1], p32[:, 2]
        s = (np.abs(x) + np.abs(y)) + np.abs(z)
        d = p32 - np.asarray(view.world_position, f32)
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        CW = view.clip_from_world.astype(f32)
        w = ((CW[3, 0] * x + CW[3, 1] * y) + CW[3, 2] * z) + CW[3, 3]
        den = np.abs(w + f32(1e-9))
    fin = np.isfinite(p32).all(1)
    tags = {"KEY_D2_INF": fin & np.isinf(d2), "KEY_DEN_WINDOW": fin & (den > 1e29) & (den < 1e31),
            "KEY_DEN_OVER": fin & (den >= 1e31), "KEY_SUM_OVERFLOW": fin & np.isinf(s), "KEY_NONFINITE": ~fin}
    return [Case("keygen_far", c, view, None, "f32", {}, tags=tags),
            Case("keygen_far_model", c, view, model_matrix("affine"), "f32", {}, tags={})]


def depth_cases(seed=0):
    """Depth colour sources.  Ordinary splats at distance 3..6, the two farthest visible ones at 40 and 12, culled ones
    (behind the camera) at 7 and 30 with the lowest and highest indices: a wrong sorted entry moves dmin or dmax by
    >= 6, i.e. the colours by > 0.1."""
    rng = np.random.default_rng(900 + seed)
    view = axis_view()
    out = []

    def mk(name, n_mid, far=(40.0, 12.0), culled=((0, 7.0), (-1, 30.0))):
        pos = list(place(view, rng.uniform(-0.6, 0.6, (n_mid, 2)), rng.uniform(3.0, 6.0, n_mid)))
        for d in far:
            pos.append(place(view, rng.uniform(-0.5, 0.5, (1, 2)), d)[0])
        pos = np.array(pos).reshape(-1, 3)
        for at, d in culled:
            p = np.array([[rng.uniform(-1, 1), rng.uniform(-1, 1), 5.0 + d]])       # behind the camera at (0, 0, 5)
            pos = np.concatenate([p, pos]) if at == 0 else np.concatenate([pos, p])
        c = cloud_of(pos, seed=seed)
        c.scale_opacity[:, :3] *= f32(0.5)
        out.append(Case(name, c, view, None, "f32", dict(rasterize_mode=B.RasterizeMode.Depth), tags={}))

    mk("depth_culled", 60)
    mk("depth_all_visible", 60, culled=())
    mk("depth_one_visible", 0, far=(9.0,))
    mk("depth_none_visible", 0, far=())
    mk("depth_two_visible", 0, far=(40.0, 12.0), culled=((0, 7.0),))
    return out


# SH basis: zeros and axes of the directions (x, y, z) in the gaussian's local frame
def _sh_directions():
    s2, s3 = math.sqrt(0.5), math.sqrt(1.0 / 3.0)
    d = [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1), (s2, s2, 0), (s2, -s2, 0), (0, s2, s2),
         (s2, 0, -s2), (s3, s3, s3), (-s3, s3, -s3), (0.6, 0.0, 0.8), (0.0, 0.8, 0.6), (0.48, 0.6, 0.64)]
    # zeros of 2zz - xx - yy (z^2 = 1/3) and of 4zz - xx - yy (z^2 = 1/5), 2zz - 3xx - 3yy (z^2 = 3/5), x^2 = 3y^2
    for z2 in (1 / 3, 1 / 5, 3 / 5):
        z = math.sqrt(z2); r = math.sqrt(1 - z2)
        d += [(r, 0, z), (0, r, -z), (r * s2, r * s2, z)]
    d += [(math.sqrt(0.75), 0.5, 0.0), (0.5, math.sqrt(0.75), 0.0)]
    return np.array(d, np.float64)


def sh_onehot_cases(seed=0):
    """48 x K gaussians, each with one non-zero SH coefficient (+-1.7), seen along the axes and the basis functions'
    zeros (one view per direction: the camera sits on the ray through the gaussian) and in general directions."""
    rng = np.random.default_rng(1000 + seed)
    gen = rng.normal(size=(8, 3))
    gen /= np.linalg.norm(gen, axis=1, keepdims=True)
    alld = np.concatenate([_sh_directions(), gen])
    # One view per direction: the eye sits at distance 4 from the gaussians' centre, opposite the wanted direction
    # (through the model's normalised columns).  The first 48 gaussians sit exactly at the centre (the direction is
    # the wanted one up to the f32 rounding of the eye and the positions); the rest within 0.05 of it.
    cases = []
    for kind in ("identity", "affine"):
        model = model_matrix(kind)
        A = np.eye(3) if model is None else model[:3, :3].astype(np.float64)
        An = A / np.linalg.norm(A, axis=0, keepdims=True)
        t = np.zeros(3) if model is None else model[:3, 3].astype(np.float64)
        for di, dl in enumerate(alld):
            wd = An @ dl
            wd /= np.linalg.norm(wd)
            centre_w = np.array([0.0, 0.0, 0.0])
            eye = centre_w - 4.0 * wd
            up = (0.0, 1.0, 0.0) if abs(wd[1]) < 0.9 else (1.0, 0.0, 0.0)
            view = B.perspective_view(tuple(eye), tuple(centre_w), 64, 48, up=up)
            n = 48 * 3
            off = np.zeros((n, 3))
            off[48:] = rng.uniform(-0.05, 0.05, (n - 48, 3))        # the first 48: exactly at the centre
            pw = centre_w + off
            Minv = np.linalg.inv(np.vstack([np.hstack([A, t[:, None]]), [0, 0, 0, 1]]))
            p = (Minv[:3, :3] @ pw.T).T + Minv[:3, 3]
            sh = np.zeros((n, 48))
            coeff = np.arange(n) % 48
            sh[np.arange(n), coeff] = np.where(np.arange(n) % 2 == 0, 1.7, -1.3)
            c = cloud_of(p, sh=sh, seed=di)
            c.scale_opacity[:, :3] = f32(0.01)
            tags = {f"SH_C{k}": coeff == k for k in range(48)}
            cases.append(Case(f"sh_{kind}_{di}", c, view, model, "f32",
                              dict(color_space=B.GaussianColorSpace.LinRec709Display), geoms=("obb3d",), tags=tags))
    return cases


def f16_specials_case(seed=0):
    """f16 layout with inf, NaN and subnormal halves in the rotation, the scale and the SH."""
    rng = np.random.default_rng(1100 + seed)
    view = off_view()
    n = 240
    pos = place(view, rng.uniform(-0.85, 0.85, (n, 2)), rng.uniform(2.0, 8.0, n))
    c = cloud_of(pos, seed=seed)
    c.scale_opacity[:, :3] *= f32(0.3)
    specials = np.array([1e5, -1e5, np.nan, 3e-6, -2e-7, 6e-8], f32)     # inf, -inf, NaN, subnormal halves
    for i in range(n):
        kind = i % 4
        v = specials[(i // 4) % len(specials)]
        if kind == 0:
            c.rotation[i, (i // 24) % 4] = v
        elif kind == 1:
            c.scale_opacity[i, (i // 24) % 3] = v
        elif kind == 2:
            c.spherical_harmonic[i, (i // 24) % 48] = v
    h = c.rounded_to_f16()
    sub = lambda a: (a != 0) & (np.abs(a) < 2.0 ** -14)
    tags = {"F16_ROT_INF": np.isinf(h.rotation).any(1), "F16_ROT_NAN": np.isnan(h.rotation).any(1),
            "F16_ROT_SUB": sub(h.rotation).any(1), "F16_SCALE_INF": np.isinf(h.scale_opacity[:, :3]).any(1),
            "F16_SCALE_NAN": np.isnan(h.scale_opacity[:, :3]).any(1), "F16_SCALE_SUB": sub(h.scale_opacity[:, :3]).any(1),
            "F16_SH_INF": np.isinf(h.spherical_harmonic).any(1), "F16_SH_NAN": np.isnan(h.spherical_harmonic).any(1),
            "F16_SH_SUB": sub(h.spherical_harmonic).any(1)}
    return Case("f16_specials", c, view, None, "f16", {}, tags=tags)


def cov_case(seed=0):
    """Precomputed-covariance records, positive definite or not: negative and zero diagonals, |c01| > sqrt(c00 c11),
    f16 inf / NaN / subnormal entries."""
    rng = np.random.default_rng(1200 + seed)
    view = off_view()
    n = 200
    pos = place(view, rng.uniform(-0.85, 0.85, (n, 2)), rng.uniform(2.0, 8.0, n))
    base = cloud_of(pos, seed=seed)
    base.scale_opacity[:, :3] *= f32(0.2)
    cov = base.precomputed_covariance()
    rot, so = cov.rotation.copy(), cov.scale_opacity.copy()
    kinds = np.arange(n) % 8
    rot[kinds == 1, 0] *= -1.0                                   # c00 < 0
    rot[kinds == 2, 1] = np.sqrt(np.abs(rot[kinds == 2, 0] * rot[kinds == 2, 3])) * 3.0     # |c01| > sqrt(c00 c11)
    rot[kinds == 3] = 0.0; so[kinds == 3, :2] = 0.0             # all zero
    rot[kinds == 4, 0] = 1e5                                    # f16 inf
    so[kinds == 5, 1] = np.nan
    rot[kinds == 6, 2] = 3e-6                                   # subnormal half
    so[kinds == 7, 0] = -so[kinds == 7, 0] - 1e-3
    raw = RawCovariance(base.position_visibility, base.spherical_harmonic, rot, so)
    h = raw.rounded_to_f16()
    c = np.concatenate([h.rotation, h.scale_opacity[:, :2]], 1)
    with np.errstate(invalid="ignore"):
        nonpd = (c[:, 0] <= 0) | (c[:, 3] <= 0) | (c[:, 5] <= 0) | (c[:, 0] * c[:, 3] - c[:, 1] ** 2 <= 0)
    tags = {"COV_NONPD": nonpd & np.isfinite(c).all(1), "COV_INF": np.isinf(c).any(1), "COV_NAN": np.isnan(c).any(1),
            "COV_SUB": ((c != 0) & (np.abs(c) < 2.0 ** -14)).any(1), "COV_PD": ~nonpd & np.isfinite(c).all(1)}
    return Case("cov_nonpd", raw, view, None, "cov", {}, geoms=("obb3d", "aabb3d"), tags=tags)


def general_cases(seed=0):
    """Ordinary clouds through the three model kinds and both views (the background every class sits in)."""
    out = []
    for kind in ("identity", "affine", "mirror"):
        for vi, view in enumerate((axis_view(), off_view())):
            rng = np.random.default_rng(1300 + seed + vi)
            n = 600
            model = model_matrix(kind)
            pos = place(view, rng.uniform(-1.0, 1.0, (n, 2)), rng.uniform(0.5, 12.0, n), model)
            c = cloud_of(pos, seed=seed + vi)
            out.append(Case(f"general_{kind}_{vi}", c, view, model, "f32", {}, tags={}))
            if kind == "affine":
                out.append(Case(f"general_f16_{vi}", c, view, None, "f16", {}, tags={}))
    return out


def case_index():
    """(name, geometries) of every case of `all_cases`, in order, without building any (test parametrisation)."""
    every = tuple(GEOMETRIES)
    two_d, three_d = ("obb2d", "aabb2d"), ("obb3d", "aabb3d")
    out = [("draw_Selected", every), ("draw_HighlightSelected", every), ("cutoff", every), ("sigma", every)]
    out += [(f"obb_{k}", every) for k in ("identity", "affine", "mirror")]
    out += [("bbox", every), ("viewport_1x48", every), ("viewport_48x1", every), ("surfel", two_d), ("surfel_extent", two_d)]
    out += [(f"sigma_zero_{v}", three_d) for v in range(10)]
    out += [("keygen_far", every), ("keygen_far_model", every)]
    out += [(n, every) for n in ("depth_culled", "depth_all_visible", "depth_one_visible", "depth_none_visible",
                                 "depth_two_visible")]
    out += [("f16_specials", every), ("cov_nonpd", three_d)]
    out += [(n, every) for n in ("general_identity_0", "general_identity_1", "general_affine_0", "general_f16_0",
                                 "general_affine_1", "general_f16_1", "general_mirror_0", "general_mirror_1")]
    n_dirs = len(_sh_directions()) + 8
    out += [(f"sh_{k}_{i}", ("obb3d",)) for k in ("identity", "affine") for i in range(n_dirs)]
    return out


@functools.lru_cache(maxsize=None)
def all_cases(oracle):
    cases = []
    cases += draw_mode_case()
    cases += cutoff_case(oracle)
    cases += sigma_case()
    cases += [obb_case(oracle, k) for k in ("identity", "affine", "mirror")]
    cases.append(bbox_case(oracle))
    cases += thin_viewport_cases()
    sc = surfel_case()
    sc.tags.update(surfel_radius_tags(oracle, sc))
    cases.append(sc)
    cases.append(surfel_extent_case())
    for c in sigma_zero_cases():
        c.tags = {"SIG0_SHORTCUT_CHANGES": shortcut_changes(oracle, c)}
        cases.append(c)
    cases += keygen_far_case()
    cases += depth_cases()
    cases.append(f16_specials_case())
    cases.append(cov_case())
    cases += general_cases()
    cases += sh_onehot_cases()
    return cases


# ---------------------------------------------------------------------------------------------------------------------
# the colour bound

# max |grad basis_k| over the unit sphere, and the sum of the magnitudes of the intermediate results each basis
# function's evaluation rounds (spherical_harmonics.wgsl:34-68 as project.cu's `sh_colour` and the oracle write it)
SH_GRAD = np.array([0, 1, 1, 1, 1, 1, 4, 1, 2, 3, 1, 6, 7.5, 6, 2, 3], np.float64)
SH_ROUND = np.array([0, 0, 0, 0, 1, 1, 7, 1, 3, 11, 2, 15, 30, 15, 7, 12], np.float64)
SHC = np.array([0.28209479177387814, -0.4886025119029199, 0.4886025119029199, -0.4886025119029199, 1.0925484305920792,
                -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396, -0.5900435899266435,
                2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658, 1.445305721320277,
                -0.5900435899266435], np.float64)


def sh_basis64(d):
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    xx, yy, zz = x * x, y * y, z * z
    return np.stack([np.ones_like(x), y, z, x, x * y, y * z, 2 * zz - xx - yy, x * z, xx - yy, y * (3 * xx - yy), x * y * z,
                     y * (4 * zz - xx - yy), z * (2 * zz - 3 * xx - 3 * yy), x * (4 * zz - xx - yy), z * (xx - yy),
                     x * (xx - 3 * yy)], 1)


def local_direction64(cloud, view, model):
    """float64 gaussian.wgsl:166-183: the normalised direction from the eye in the model's normalised column frame."""
    A = np.eye(3) if model is None else model[:3, :3].astype(np.float64)
    t = np.zeros(3) if model is None else model[:3, 3].astype(np.float64)
    p = cloud.position_visibility[:, :3].astype(np.float64)
    with np.errstate(all="ignore"):
        pw = p @ A.T + t
        d = pw - np.asarray(view.world_position, np.float64)
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        An = A / np.linalg.norm(A, axis=0, keepdims=True)
        loc = d @ An
        return loc / np.linalg.norm(loc, axis=1, keepdims=True)


def colour_bound(cloud, view, model, color_space: int, ids=None, eps_dir=None):
    """(n, 3) bound on |CUDA colour - oracle colour| of each record (RasterizeMode::Color), from the float64
    direction and the (decoded) SH coefficients of the gaussian.

    * Direction: the kernel normalises with rsqrt.approx (<= 2 ulp, 4 U relative) times a rounded multiply, the
      oracle with an IEEE sqrt and a division (2 U).  An identity model normalises twice (the eye direction, then the
      local one), others three times with a rounded dot product between: the unit direction the SH sees differs by
      eps_dir <= 16 U (identity) or 48 U (others) in each component.  A basis function moves by at most its gradient
      bound times sqrt(3) eps_dir, plus the roundings of its own evaluation on both sides (2 U times the sum of
      its intermediate magnitudes).
    * Constants and accumulation: the kernel folds c_shc into the basis (one rounding) and accumulates with fma (one
      rounding per step); the oracle rounds (shc * sh) * basis (two) and each add (one): 4 U |term| per term, and
      2 x 16 rounding steps of a partial sum bounded by 0.5 + sum |term|.
    * sRGB (color_space 0): v / 12.92 against v * (1 / 12.92) (2 U relative plus the input error / 12.92), and
      __powf = ex2.approx(2.4 lg2.approx(x)): lg2 within 2^-22.6 absolute plus a rounding of 2.4 lg2 x, ex2 within
      2 ulp: <= 1e-6 + 4e-7 |log2 x| relative (2x margin), plus 2.4 out / x times the input error.
    Records with a non-finite coefficient or direction get bound 0: their colours must be the same value or both
    NaN."""
    if ids is not None:
        cloud = B.PlanarGaussian3d(*(getattr(cloud, k)[ids] for k in ("position_visibility", "spherical_harmonic",
                                                                          "rotation", "scale_opacity")))
    if eps_dir is None:
        eps_dir = (16.0 if model is None else 48.0) * U
    dl = local_direction64(cloud, view, model)
    basis = sh_basis64(dl)                                          # (n, 16)
    sh = cloud.spherical_harmonic.astype(np.float64).reshape(-1, 16, 3)
    with np.errstate(all="ignore"):
        term = np.abs(sh) * np.abs(SHC)[None, :, None]              # |sh shc|
        per = term * (SH_GRAD[None, :, None] * math.sqrt(3.0) * eps_dir + 2 * U * SH_ROUND[None, :, None]
                      + 4 * U * np.abs(basis)[:, :, None])
        tsum = (term * np.abs(basis)[:, :, None]).sum(1)           # sum |term|
        dv = per.sum(1) + 32 * U * (0.5 + tsum)
        v = 0.5 + (sh * SHC[None, :, None] * basis[:, :, None]).sum(1)
        if color_space == 0:
            x = (v + 0.055) / 1.055
            out = np.where(v <= 0.04045, v / 12.92, np.abs(x) ** 2.4)
            lin = dv / 12.92 + 2 * U * np.abs(out)
            kp = 1e-6 + 4e-7 * np.abs(np.log2(np.where(x > 0, x, 1.0)))
            pw = 2.4 * out / np.where(x > 0, x, 1.0) * (dv / 1.055 + 3 * U * np.abs(x)) + kp * out
            b = np.where(v <= 0.04045, lin, pw)
            near = np.abs(v - 0.04045) <= dv + 1e-7                  # the two sides may take different branches
            b = np.where(near, np.maximum(lin, pw) + 2e-7, b)
        else:
            b = dv
    finite = np.isfinite(dl).all(1)[:, None] & np.isfinite(sh).all(1) & np.isfinite(b)
    return np.where(finite, b, 0.0)


def colours_agree(got, want, bound):
    """Per component: equal, both NaN, or within the bound."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    with np.errstate(invalid="ignore"):
        return (got == want) | (np.isnan(got) & np.isnan(want)) | (np.abs(got - want) <= bound)


def bits_agree(got, want):
    """f32 arrays equal bit for bit (the sign of a zero counted), NaN compared as a class: a NaN's payload is not part
    of the result (x86 makes 0xFFC00000, CUDA 0x7FFFFFFF)."""
    got, want = np.asarray(got, f32), np.asarray(want, f32)
    return (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
