"""Gaussian4d inputs built to reach each part of the reference's 4D rule, and the f32 error bounds the record and colour
checks of tests/test_wgsl_restatement_4d.py and tests/test_gpu_temporal_wgsl.py hold the port to.

The bounds: a running error analysis of bgs_render_4d's f32 evaluation (include/bgs.h, rule 1-7, in the order the
header writes it).  `E` carries a float64 value and a bound on how far an f32 evaluation of the same expression, in the
same order, can be from that value.  With u = 2^-24 (the unit roundoff of round-to-nearest binary32) each operation
adds u |result| to the propagated input errors, by the first-order rules with their second-order terms kept:

  a +- b:  ea + eb                          a * b:  |a| eb + |b| ea + ea eb
  a / b:   (ea + |a / b| eb) / (|b| - eb)   sqrt a: sqrt(a + ea) - sqrt(max(a - ea, 0))

so a bound is always a multiple of u times the magnitudes of the terms that produce the value, never a number fitted to
an observed error.  The float64 values carry their own rounding, 2^-52 relative per step, which is 2^-28 of the f32 unit
and is covered by adding 2^-40 |value| to each final bound (`E.bound`).  Library functions enter with their documented
accuracy:
  * det_exp: 1/2 ulp (u |result|) after an f64 series whose own error is below 2^-50;
  * det_cos: DET_COS_ERR(x) (include/bgs.h rule 7, derived in det_cos_bound);
  * the oracle's std::pow (sRGB decode) and std::sqrt: correctly rounded to within 1 ulp (2u relative);
  * the kernel's colour path (gpu=True): rsqrt.approx.f32 relative error <= 2^-22 (2 ulp) for each normalisation,
    __powf = ex2.approx(2.4 * lg2.approx(x)) with lg2's absolute error <= 2^-22 and ex2's relative error <= 2^-22
    (PTX ISA), and FMA sums, whose one rounding per step is covered by the unfused bound's two.
"""
from __future__ import annotations

import math

import numpy as np

import bevy_gaussian_splatting_b200 as B

f32 = np.float32
U = 2.0 ** -24
SHC = [0.28209479177387814, -0.4886025119029199, 0.4886025119029199, -0.4886025119029199, 1.0925484305920792,
       -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396, -0.5900435899266435,
       2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658, 1.445305721320277,
       -0.5900435899266435]
# det_cos (include/bgs.h rule 7): r = x - k C, C = 6.283185307179586 = 2 pi - 2.4493e-16; the product k C is rounded
# once in f64 (1/2 ulp <= 2^-53 |k C|) and the subtraction is exact (Sterbenz), so |r - (x - 2 pi k)| <= |x| (2^-53 +
# 2.4493e-16 / 2 pi) (1 + 2^-52) = |x| 1.5005e-16.  cos is 1-Lipschitz; the degree-36 series and its f64 Horner sum add
# below 1e-15 for |r| <= pi + 1; the f32 rounding of the result adds 1/2 ulp <= 2^-25.
TWO_PI_MINUS_C = 2.4492935982947064e-16         # 2 pi - 6.283185307179586 (2 pi to 40 digits, less the f64 constant)
DET_COS_SLOPE = (2.0 ** -53 + TWO_PI_MINUS_C / (2 * math.pi)) * (1 + 2.0 ** -52)
DET_COS_RANGE = 2.0 ** 53                      # |x| up to here: |r| <= pi + |x| DET_COS_SLOPE <= pi + 1.4


def det_cos_bound(x):
    """|det_cos(x) - cos(x)| for the f32 argument x, |x| <= DET_COS_RANGE."""
    return abs(x) * DET_COS_SLOPE + 1e-15 + 2.0 ** -25


class E:
    """A float64 value and a bound on the f32 evaluation's distance from it."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=0.0):
        self.v, self.e = float(v), float(e)

    @staticmethod
    def of(x):
        return x if isinstance(x, E) else E(x)

    def _r(self, v, e):
        return E(v, e + U * abs(v))

    def __add__(self, o):
        o = E.of(o); return self._r(self.v + o.v, self.e + o.e)

    __radd__ = __add__

    def __sub__(self, o):
        o = E.of(o); return self._r(self.v - o.v, self.e + o.e)

    def __rsub__(self, o):
        return E.of(o) - self

    def __neg__(self):
        return E(-self.v, self.e)

    def __mul__(self, o):
        o = E.of(o); return self._r(self.v * o.v, abs(self.v) * o.e + abs(o.v) * self.e + self.e * o.e)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = E.of(o)
        if abs(o.v) <= o.e:
            return E(self.v / o.v if o.v else math.inf, math.inf)
        q = self.v / o.v
        return self._r(q, (self.e + abs(q) * o.e) / (abs(o.v) - o.e))

    def __rtruediv__(self, o):
        return E.of(o) / self

    def sqrt(self, rel=U):
        r = math.sqrt(max(self.v, 0.0))
        e = math.sqrt(max(self.v, 0.0) + self.e) - math.sqrt(max(self.v - self.e, 0.0))
        return E(r, e + rel * r)

    def rel(self, rel):
        """The value times (1 + d), |d| <= rel: an approximate operation's documented relative error."""
        return E(self.v, self.e * (1 + rel) + rel * abs(self.v))

    @property
    def bound(self):
        return self.e + 2.0 ** -40 * abs(self.v)


def K(c):
    """A literal of the WGSL (float64 here) as the f32 constant the port uses: its rounding is the error."""
    return E(c, abs(float(f32(c)) - c))


def emax(a, b):
    a, b = E.of(a), E.of(b)
    return E(max(a.v, b.v), max(a.e, b.e))


def emin(a, b):
    a, b = E.of(a), E.of(b)
    return E(min(a.v, b.v), max(a.e, b.e))


def mat4_point(m16, p):
    """((m0 x + m1 y) + m2 z) + m3 per row, m 16 floats column-major (bgs.h's order)."""
    return [((m16[r] * p[0] + m16[4 + r] * p[1]) + m16[8 + r] * p[2]) + m16[12 + r] for r in range(4)]


def condition(gs, q8, so, tt, t):
    """include/bgs.h rules 3-5 on E: cov_t, c12, cov3d (6), delta_mean (3), the exponent and marginal_t."""
    dt = E(t) - E(tt[0])
    sd = [E(gs) * so[0], E(gs) * so[1], E(gs) * so[2], E(tt[1])]
    w, x, y, z, wr, xr, yr, zr = (E(v) for v in q8)
    Ml = [[w, -x, -y, -z], [x, w, -z, y], [y, z, w, -x], [z, -y, x, w]]
    Mr = [[wr, -xr, -yr, -zr], [xr, wr, zr, -yr], [yr, -zr, wr, xr], [zr, yr, -xr, wr]]
    M = [[(((Mr[0][r] * Ml[c][0] + Mr[1][r] * Ml[c][1]) + Mr[2][r] * Ml[c][2]) + Mr[3][r] * Ml[c][3]) * sd[c]
          for r in range(4)] for c in range(4)]
    sig = lambda c, r: ((M[r][0] * M[c][0] + M[r][1] * M[c][1]) + M[r][2] * M[c][2]) + M[r][3] * M[c][3]  # noqa: E731
    cov_t = sig(3, 3)
    q = ((E(-0.5) * dt) * dt) / cov_t
    m = math.exp(q.v) if q.v > -745 else 0.0
    marginal = E(m, m * (math.expm1(q.e) if q.e < 700 else math.inf) + U * m)
    c12 = [sig(0, 3), sig(1, 3), sig(2, 3)]
    cond = lambda c, r: sig(c, r) - (c12[c] * c12[r]) / cov_t  # noqa: E731
    c3 = [cond(0, 0), cond(0, 1), cond(0, 2), cond(1, 1), cond(1, 2), cond(2, 2)]
    dm = [(c12[i] / cov_t) * dt for i in range(3)]
    return dict(dt=dt, cov_t=cov_t, c12=c12, c3=c3, dm=dm, q=q, marginal=marginal)


def ndc(clip16, pw):
    c = mat4_point(clip16, pw)
    den = c[3] + K(0.000000001)
    return [c[i] / den for i in range(3)]


def geometry(view, W, H, pw, c3, cutoff, aabb):
    """helpers.wgsl:8-119 in bgs.h's order on the conditioned covariance at pw (E): the record's fields 2-5 and the
    half extents (hx, hy) of the pixel bbox."""
    vfw = [float(x) for x in view.view_from_world]
    cfv = [float(x) for x in view.clip_from_view]
    Vrk = [[c3[0], c3[1], c3[2]], [c3[1], c3[3], c3[4]], [c3[2], c3[4], c3[5]]]
    t = mat4_point(vfw, pw)
    fx, fy = E(cfv[0]) * W, E(cfv[5]) * H
    sz = 1.0 / (t[2] * t[2])
    J00, J20 = fx / t[2], -(fx * t[0]) * sz
    J11, J21 = -fy / t[2], (fy * t[1]) * sz
    Tm = [[vfw[i * 4 + 0] * J00 + vfw[i * 4 + 2] * J20, vfw[i * 4 + 1] * J11 + vfw[i * 4 + 2] * J21] for i in range(3)]
    Y = [[(Vrk[i][0] * Tm[0][b] + Vrk[i][1] * Tm[1][b]) + Vrk[i][2] * Tm[2][b] for b in range(2)] for i in range(3)]
    a = ((Tm[0][0] * Y[0][0] + Tm[1][0] * Y[1][0]) + Tm[2][0] * Y[2][0]) + K(0.3)
    b = (Tm[0][1] * Y[0][0] + Tm[1][1] * Y[1][0]) + Tm[2][1] * Y[2][0]
    c = ((Tm[0][1] * Y[0][1] + Tm[1][1] * Y[1][1]) + Tm[2][1] * Y[2][1]) + K(0.3)
    det = a * c - b * b
    mid = 0.5 * (a + c)
    term = emax(0.0, mid * mid - det).sqrt()
    l1 = mid + term
    if aabb:
        l2 = emax(mid - term, 0.0)
        Rq = cutoff * emax(l1.sqrt(), l2.sqrt())
        dinv = 1.0 / det
        h = 0.5 * Rq
        return dict(fields=[c * dinv, -b * dinv, a * dinv, Rq], hx=h, hy=h, cov2d=(a, b, c))
    aa = (a - c) * (a - c)
    bb = (aa + (4.0 * b) * b).sqrt()
    major = (((a + c) + bb) * 0.5).sqrt()
    minor = (((a + c) - bb) * 0.5).sqrt()
    Bx, By = cutoff * major, cutoff * minor
    evx, evy = -b, l1 - a
    el = (evx * evx + evy * evy).sqrt()
    e1x, e1y = evx / el, evy / el
    e2x, e2y = e1y, -e1x
    fields = [(2.0 * e1x) / Bx, (-2.0 * e1y) / Bx, (2.0 * e2x) / By, (-2.0 * e2y) / By]
    ab = lambda q: E(abs(q.v), q.e)  # noqa: E731
    hx = 0.5 * (ab(e1x) * Bx + ab(e2x) * By)
    hy = 0.5 * (ab(e1y) * Bx + ab(e2y) * By)
    return dict(fields=fields, hx=hx, hy=hy, cov2d=(a, b, c))


def normalize3(a, gpu):
    if gpu:    # rsqrt.approx: one approximate reciprocal square root, three products
        inv = (((a[0] * a[0] + a[1] * a[1]) + a[2] * a[2]).sqrt(rel=0.0))
        inv = (1.0 / inv).rel(2.0 ** -22)
        inv = E(inv.v, inv.e - U * abs(inv.v))           # (rsqrt is one operation: no separate division rounding)
        return [x * inv for x in a]
    n = ((a[0] * a[0] + a[1] * a[1]) + a[2] * a[2]).sqrt()
    return [x / n for x in a]


def srgb(v, gpu):
    """spherical_harmonics.wgsl's decode; a value within its error of the branch point 0.04045 gets an infinite bound."""
    if abs(v.v - 0.04045) <= v.e:
        return E(v.v, math.inf)
    if v.v <= 0.04045:
        return v / K(12.92) if not gpu else v * E(1.0 / 12.92, 2 * U / 12.92)
    x = (v + K(0.055)) / K(1.055) if not gpu else (v + K(0.055)) * E(1.0 / 1.055, 2 * U / 1.055)
    p = x.v ** 2.4
    dp = p * ((1 + x.e / x.v) ** 2.4 - 1)          # x^2.4's change over the input error, exactly
    if gpu:   # ex2(2.4 lg2 x): lg2's absolute error and the product's rounding enter the exponent; then ex2's error
        arg_err = 2.4 * 2.0 ** -22 + U * abs(2.4 * math.log2(x.v))
        return E(p, dp + p * (2.0 ** arg_err - 1.0) * (1 + 2.0 ** -22) + 2.0 ** -22 * p)
    return E(p, dp + 2 * U * p)


def spherindrical(view, transform16, pw, dt, duration, sh, color_space, gpu=False, classes=None):
    """rule 7's colour at pw (E) for dt, duration (f32 values), sh (144): -> 3 E."""
    cam = [float(x) for x in view.world_position]
    dlt = [pw[i] - cam[i] for i in range(3)]
    dw = normalize3(dlt, gpu)
    loc = []
    for c in range(3):
        bn = normalize3([E(transform16[c * 4 + i]) for i in range(3)], gpu)
        loc.append((bn[0] * dw[0] + bn[1] * dw[1]) + bn[2] * dw[2])
    x, y, z = normalize3(loc, gpu)
    xx, yy, zz = x * x, y * y, z * z
    basis = [E(1.0), y, z, x, x * y, y * z, (2.0 * zz - xx) - yy, x * z, xx - yy, y * (3.0 * xx - yy), (x * y) * z,
             y * ((4.0 * zz - xx) - yy), z * ((2.0 * zz - 3.0 * xx) - 3.0 * yy), x * ((4.0 * zz - xx) - yy), z * (xx - yy),
             x * (xx - 3.0 * yy)]
    basis = [K(SHC[k]) * basis[k] for k in range(16)]
    theta = E(float(f32(f32(dt) / f32(duration))))       # the f32 theta itself: exact input to the argument
    out = []
    args = [float(f32(f32(2.0 * float(f32(math.pi))) * f32(theta.v))), float(f32(f32(4.0 * float(f32(math.pi))) * f32(theta.v)))]
    tcos = [E(math.cos(a), det_cos_bound(a)) for a in args]
    for ch in range(3):
        acc = [E(0.5), E(0.0), E(0.0)]
        for blk in range(3):
            for k in range(16):
                acc[blk] = acc[blk] + basis[k] * float(sh[48 * blk + 3 * k + ch])
        rgb = (acc[0] + tcos[0] * acc[1]) + tcos[1] * acc[2]
        out.append(srgb(rgb, gpu) if color_space == 0 else rgb)
    return out


# ---------------------------------------------------------------- inputs
def ulp_walk(x, steps):
    return (np.asarray([x], np.float32).view(np.int32).astype(np.int64) + np.asarray(list(steps))).astype(np.int32).view(np.float32)


def unit_rot(rng, n):
    q = rng.normal(size=(n, 4))
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def edge_cloud(n=64, seed=0, spread=1.2, center=(0.0, 0.0, 0.0)):
    """A PlanarGaussian4d of n gaussians around `center`, each row built to reach one part of the rule:
      rows 0 mod 8: random rotation pairs with norms 0.5 to 2 (every row's pair is unnormalised).  They do not couple
        space and time: M_l and M_r are each |q| times an orthogonal matrix, so transpose(M) * M = |q|^2 |q_r|^2 S^2 is
        diagonal, c12 = 0 and delta_mean = 0 in exact arithmetic for every row (DESIGN.md, Gaussian4d).  The port's
        f32 delta_mean is rounding noise held to its E bound, and every Velocity is 0: the Velocity checks here cover
        the culling and the zero colour and opacity only;
      1 mod 8: dt = 0 (timestamp = `time` of the frame, 0.5);
      2 mod 8: marginal_t within a few ulps of 0.05 (timescale ulp-walked around dt / sqrt(2 ln 20));
      3 mod 8: tiny cov_t (timescale 1e-3, |dt| <= 2e-4): delta_mean is a large ratio of small numbers;
      4 mod 8: only the spatial SH block non-zero; 5: only the cos(2 pi theta) block; 6: only the cos(4 pi theta) block;
      7 mod 8: all three blocks, timestamps making theta = 0, +-1/4, +-1/2, 1 and 37.3 for the window (0, 1).
    Visibility is a mix of 0, 1 and class labels; opacities span 0.05 to 0.95.  One scale axis is 4x the others: the
    OBB quad of a near-isotropic footprint turns with its f32 eigenvector, so its pixel bbox is not decided by the rule."""
    rng = np.random.default_rng(seed)
    pos = (rng.random((n, 3)) - 0.5) * 2 * spread + np.asarray(center)
    vis = rng.choice(np.array([0.0, 1.0, 2.0, 3.5]), n)
    q1, q2 = unit_rot(rng, n), unit_rot(rng, n)
    norms = rng.uniform(0.5, 2.0, (n, 2))
    rot8 = np.concatenate([q1 * norms[:, :1], q2 * norms[:, 1:]], 1)
    so = np.concatenate([rng.uniform(0.02, 0.04, (n, 3)), rng.uniform(0.05, 0.95, (n, 1))], 1)
    so[np.arange(n), rng.integers(0, 3, n)] *= 4.0     # anisotropic footprints: a well-conditioned eigenvector
    tt = np.zeros((n, 4))
    tt[:, 0] = rng.uniform(0.2, 0.8, n)
    tt[:, 1] = rng.uniform(0.4, 1.2, n) * rng.choice([-1.0, 1.0], n)
    sh = rng.normal(0, 0.25, (n, 144))
    thetas = [0.0, 0.25, -0.25, 0.5, -0.5, 1.0, 37.3]
    for i in range(n):
        kind = i % 8
        if kind == 1:
            tt[i, 0] = 0.5
        elif kind == 2:
            dt = 0.5 - tt[i, 0]
            st0 = abs(dt) / math.sqrt(2 * math.log(20.0))
            tt[i, 1] = float(ulp_walk(st0, [(i // 8) % 9 - 4])[0])
            rot8[i] = [1, 0, 0, 0, 1, 0, 0, 0]           # cov_t = timescale^2 exactly: the walk steps marginal_t
        elif kind == 3:
            tt[i, 1] = 1e-3
            tt[i, 0] = 0.5 + rng.uniform(-2e-4, 2e-4)
        elif kind in (4, 5, 6):
            blk = kind - 4
            keep = sh[i, 48 * blk:48 * blk + 48].copy()
            sh[i] = 0.0
            sh[i, 48 * blk:48 * blk + 48] = keep * 2
        elif kind == 7:
            tt[i, 0] = 0.5 - thetas[(i // 8) % len(thetas)]
    c = B.PlanarGaussian4d(np.concatenate([pos, vis[:, None]], 1).astype(np.float32), sh.astype(np.float32),
                           rot8.astype(np.float32), so.astype(np.float32), tt.astype(np.float32))
    return c


def theta_cloud(thetas, seed=1, center=(0.0, 0.0, 0.0)):
    """One visible gaussian per theta (window (0, 1), time 0.5: timestamp = 0.5 - theta, timescale 1e9 so that the time
    mask passes at any dt), only the time blocks non-zero: the colour is 0.5 + t1 s1 + t2 s2."""
    rng = np.random.default_rng(seed)
    n = len(thetas)
    pos = np.asarray(center) + (rng.random((n, 3)) - 0.5) * 0.8
    sh = np.zeros((n, 144))
    sh[:, 48:] = rng.normal(0, 0.2, (n, 96))
    rot8 = np.tile([1.0, 0, 0, 0, 1.0, 0, 0, 0], (n, 1))
    so = np.tile([0.05, 0.04, 0.03, 0.8], (n, 1))
    tt = np.zeros((n, 4))
    tt[:, 0] = 0.5 - np.asarray(thetas, np.float64)
    tt[:, 1] = 1e9
    return B.PlanarGaussian4d(np.concatenate([pos, np.ones((n, 1))], 1).astype(np.float32), sh.astype(np.float32),
                              rot8.astype(np.float32), so.astype(np.float32), tt.astype(np.float32))


def model_matrix():
    """A rotated, non-uniformly scaled, sheared, translated model matrix (4x4 row-major float32).  The shear makes its
    columns non-orthogonal: world_to_local_direction's final normalize then changes the direction (with orthogonal
    columns the dot products with the normalised columns already have unit length)."""
    a, b = 0.6, -0.35
    ry = np.array([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]])
    rx = np.array([[1, 0, 0], [0, math.cos(b), -math.sin(b)], [0, math.sin(b), math.cos(b)]])
    m = np.eye(4, dtype=np.float32)
    m[:3, :3] = (ry @ rx @ np.diag([1.25, 0.8, 1.1]) @ np.array([[1, 0.35, 0], [0, 1, 0], [0.2, 0, 1]])).astype(np.float32)
    m[:3, 3] = [0.3, -0.2, 0.4]
    return m


def off_axis_view(w, h):
    """The eye off every axis, the target not the origin, the up vector tilted."""
    return B.perspective_view((2.2, 1.8, 4.5), (0.1, 0.05, -0.2), w, h, up=(0.15, 1.0, -0.05))


def clamp_e(x, lo, hi):
    return emin(emax(x, lo), hi)


def hsv_e(h, sat, v):
    """Bevy's hsv_to_rgb on E (k = (base + h / FRAC_PI_3) % 6).  max(0, min(k, min(4 - k, 1))) is 0 on both sides of a
    multiple of 6, so the wrap of % adds no error: k carries x's."""
    out = []
    for base in (5.0, 3.0, 1.0):
        x = base + h / K(math.pi / 3.0)
        k = x - 6.0 * math.trunc(x.v / 6.0)
        out.append(v - v * sat * emax(0.0, emin(k, emin(4.0 - k, 1.0))))
    return out


def depth_rgb_e(depth, dmin, dmax):
    """material/depth.wgsl:3-11 on E (bgs.h rule 7's Depth colour)."""
    def smooth(e0, e1, x):
        t = clamp_e((x - e0) / (e1 - e0), 0.0, 1.0)
        return (t * t) * (3.0 - 2.0 * t)
    nd = clamp_e((depth - dmin) / (dmax - dmin), 0.0, 1.0)
    return [smooth(0.5, 1.0, nd), 1.0 - (E(abs(nd.v - 0.5), nd.e) * 2.0), 1.0 - smooth(0.0, 0.5, nd)]


def flow_rgb_e(clip16, prev16, pw, p0, delta_time):
    """optical_flow.wgsl on E: the clip of the moved p, the previous clip of the unmoved p0; atan2 is the port's fixed
    series rounded to f32 (u |angle|) on the rounded flow; an angle within its error of 0 is undecided."""
    c, cp = mat4_point(clip16, pw), mat4_point(prev16, p0)
    mvx = (c[0] / c[3] - cp[0] / cp[3]) * 0.5
    mvy = (c[1] / c[3] - cp[1] / cp[3]) * -0.5
    fx, fy = mvx / E(delta_time), mvy / E(delta_time)
    radius = (fx * fx + fy * fy).sqrt()
    r2 = fx.v * fx.v + fy.v * fy.v
    ang = math.atan2(fy.v, fx.v)
    ea = (abs(fx.v) * fy.e + abs(fy.v) * fx.e) / max(r2 - fx.e * fx.e - fy.e * fy.e, 1e-300) + U * abs(ang)
    if abs(ang) <= ea or r2 == 0.0:
        return [E(0.0, math.inf)] * 3
    angle = E(ang, ea)
    if ang < 0:
        angle = angle + K(2 * math.pi)
    return hsv_e(angle, clamp_e(radius, 0.0, 1.0), E(1.0))


# ---------------------------------------------------------------- records against the emulator
MODE_NAMES = {B.RasterizeMode.Color: "color", B.RasterizeMode.Depth: "depth", B.RasterizeMode.Position: "position",
              B.RasterizeMode.Classification: "classification", B.RasterizeMode.OpticalFlow: "optical_flow",
              B.RasterizeMode.Velocity: "velocity"}


def shader_for(view, u, s, window, extras=None):
    from wgsl_emu import CloudU, ViewU, mat4x4
    from wgsl_emu_4d import Shader4d
    prev = dt = None
    nc = int(s.num_classes)
    if extras is not None:
        prev = mat4x4(*[float(x) for x in extras.previous_clip_from_world])
        dt, nc = float(extras.delta_time), int(extras.num_classes)
    return Shader4d(ViewU(view.to_abi()), CloudU(u), float(u.time), window[0], window[1], use_obb=not s.aabb,
                    adaptive=s.opacity_adaptive_radius, rasterize=MODE_NAMES[s.rasterize_mode], prev_clip_from_world=prev,
                    delta_time=dt, num_classes=nc)


def _bbox_decision(c, h, lim):
    """set_bbox's integer edges from a centre and half extent (E): (lo, hi, margin over bound), bgs.h's slack rule."""
    sl = h.v * 1e-3 + 1e-2
    a = (c.v - h.v) - (0.5 + sl)
    b = (c.v + h.v) - (0.5 - sl)
    err = c.e + h.e * (1 + 1e-3) + 4 * U * (abs(c.v) + abs(h.v) + 1)
    lo, hi = math.ceil(a), math.floor(b)
    margin = min(abs(a - round(a)), abs(b - round(b)))
    return max(lo, 0), min(hi, lim - 1), lo <= hi and max(lo, 0) <= min(hi, lim - 1), margin > err, min(1.0, 4 * err)


def _frustum_margin(n3):
    """The base frustum test on E ndc: (in, decided)."""
    inside = abs(n3[0].v) < 1.1 and abs(n3[1].v) < 1.1 and abs(n3[2].v - 0.5) < 0.5
    decided = all(abs(abs(v.v) - 1.1) > v.bound for v in n3[:2]) and abs(abs(n3[2].v - 0.5) - 0.5) > n3[2].bound
    return inside, decided


def check_records(rec, ids, cloud, view, u, s, window, sorted_ids, extras=None, gpu=False, bounds=None):
    """Hold records (bgs_debug_projected's layout, by front-to-back rank) to the emulator: every decision equal
    unless its float64 margin is inside the E bound; every value within its E bound.  The base frustum test is checked
    both ways: `ids` must be exactly the gaussians of `cloud` the emulator keeps at their base position, those within
    their error of a frustum plane aside.  -> (compared, undecided, expected): `expected` is the number of undecided
    records the bounds predict -- each of the two edge arguments of a bbox axis lies within its error of an integer
    with probability 2 err, and each row built on the time threshold counts 1.
    `bounds` (a dict), when given, receives per drawn gaussian index the E bounds of its record's centre (2), fields 2-5
    (4), colour (3) and opacity, or None for an undecided one: the frame check carries them through the blend."""
    sh4 = shader_for(view, u, s, window, extras)
    W, H = int(view.width), int(view.height)
    T16 = [float(x) for x in u.transform]
    clip16 = [float(x) for x in view.to_abi().clip_from_world]
    hw, hh = 0.5 * W, 0.5 * H
    draw_sel = s.draw_mode == B.DrawMode.Selected
    highlight = s.draw_mode == B.DrawMode.HighlightSelected
    n = len(cloud)
    if sh4.rasterize == "depth":
        sh4.depth_entries = tuple(
            __import__("wgsl_emu").Vec(*cloud.position_visibility[int(sorted_ids[i]), :3].tolist()) for i in (1, n - 1))
    duration = float(f32(f32(window[1]) - f32(window[0])))
    compared = undecided = 0
    expected = 0.0
    listed = set(int(i) for i in ids)
    for gi in range(n):
        if gi in listed:
            continue
        n0 = ndc(clip16, mat4_point(T16, [E(float(x)) for x in cloud.position_visibility[gi, :3]])[:3])
        inside, decided = _frustum_margin(n0)
        assert not (inside and decided), (gi, "the emulator keeps a gaussian at its base that the port culls")
    for r, gi in enumerate(ids):
        gi = int(gi)
        pv = [float(x) for x in cloud.position_visibility[gi]]
        so = [float(x) for x in cloud.scale_opacity[gi]]
        q8 = [float(x) for x in cloud.isotropic_rotations[gi]]
        tt = [float(x) for x in cloud.timestamp_timescale[gi]]
        shv = cloud.spherindrical_harmonic[gi]
        vs = sh4.vs_points_4d(__import__("wgsl_emu").Vec(*pv[:3]), [float(x) for x in shv], q8, so, tt, visibility=pv[3],
                              draw_selected=draw_sel, highlight_selected=highlight)
        o = rec[r]
        bb = o[6:8].view(np.uint32)
        got_drawn = (bb[0] & 0xFFFF) <= (bb[0] >> 16)
        pw0 = mat4_point(T16, [E(x) for x in pv[:3]])
        n0 = ndc(clip16, pw0[:3])
        base_c = (n0[0] * hw + hw, hh - n0[1] * hh)
        assert vs["reason"] != "base" or any(abs(abs(v.v) - 1.1) <= v.bound for v in n0[:2]) or \
            abs(abs(n0[2].v - 0.5) - 0.5) <= n0[2].bound, (gi, "the port keeps a gaussian the emulator culls at its base")
        ok = True
        if vs["reason"] in (None, "moved", "mask"):
            g = condition(float(u.global_scale), q8, so, tt, float(u.time))
            if abs(g["marginal"].v - 0.05) <= g["marginal"].bound:
                ok = False
                expected += 1        # (edge rows 2 mod 8 are built within a few ulps of the threshold)
        if vs["reason"] in (None, "moved"):
            pm = mat4_point(T16, [E(pv[i]) + g["dm"][i] for i in range(3)])
            nm = ndc(clip16, pm[:3])
            ok &= all(abs(abs(v.v) - 1.1) > v.bound for v in nm[:2]) and abs(abs(nm[2].v - 0.5) - 0.5) > nm[2].bound
        if vs["reason"] is not None:
            if not ok:
                undecided += 1
                if bounds is not None:
                    bounds[gi] = None
                continue
            assert not got_drawn and o[8] == 0 and o[9] == 0 and o[10] == 0, (gi, vs["reason"], o)
            assert o[11] == f32(f32(so[3]) * f32(u.global_opacity)), (gi, o[11])
            for k in range(2):
                assert abs(o[k] - base_c[k].v) <= base_c[k].bound, (gi, k, o[k], base_c[k].v, base_c[k].bound)
            compared += 1
            continue
        cm = (nm[0] * hw + hw, hh - nm[1] * hh)
        geo = geometry(view.to_abi(), W, H, pm[:3], g["c3"], E(vs["cutoff"], 4 * U * vs["cutoff"]), s.aabb)
        # the emulator's own half extents: the emitted corners' largest pixel offset
        from wgsl_emu import ndc_to_pixel
        P = np.array([ndc_to_pixel(v["position"].xy.v, W, H) for v in vs["vertices"]])
        c_px = ndc_to_pixel(vs["projected_position"].xy.v, W, H)
        hx = E(np.abs(P[:, 0] - c_px[0]).max(), geo["hx"].e)
        hy = E(np.abs(P[:, 1] - c_px[1]).max(), geo["hy"].e)
        bx = _bbox_decision(E(c_px[0], cm[0].e), hx, W)
        by = _bbox_decision(E(c_px[1], cm[1].e), hy, H)
        expected += min(1.0, bx[4] + by[4])
        opac = E(so[3]) * g["marginal"]
        rgb = None
        if sh4.rasterize == "velocity":
            fut = condition(float(u.global_scale), q8, so, tt, float(f32(f32(u.time) + f32(1e-3))))
            fm = fut["marginal"]
            ok &= abs(fm.v - 0.05) > fm.bound
            fdm = fut["dm"] if fm.v > 0.05 else [E(0.0)] * 3
            v = [(fdm[i] - g["dm"][i]) / K(1e-3) for i in range(3)]
            ln = ((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]).sqrt()
            sc = (ln - 1.0)
            ok &= abs(sc.v - 1e-2) > sc.bound and abs(sc.v) > sc.bound
        if not ok:
            undecided += 1
            if bounds is not None:
                bounds[gi] = None
            continue
        bbox_decided = bx[3] and by[3]     # (an undecided bbox edge lies the slack outside the quad: values still compare)
        undecided += not bbox_decided
        want_drawn = bx[2] and by[2]
        assert got_drawn == want_drawn or not bbox_decided, (gi, got_drawn, bx, by)
        if want_drawn and bbox_decided:
            assert (int(bb[0] & 0xFFFF), int(bb[0] >> 16), int(bb[1] & 0xFFFF), int(bb[1] >> 16)) == (bx[0], bx[1], by[0], by[1]), \
                (gi, bb, bx, by)
        for k in range(2):
            assert abs(o[k] - c_px[k]) <= cm[k].bound, (gi, k, o[k], c_px[k], cm[k].bound)
        if s.aabb:
            want = list(vs["conic"].v) + [abs(vs["vertices"][3]["bb"].z)]
        else:
            Pm = P - c_px
            A = np.stack([0.5 * (Pm[2] - Pm[0]), 0.5 * (Pm[1] - Pm[0])], axis=1)
            want = list(np.linalg.inv(A).ravel())
        for k in range(4):
            assert abs(o[2 + k] - want[k]) <= geo["fields"][k].bound, (gi, k, o[2 + k], want[k], geo["fields"][k].bound)
        col = vs["color"]
        if bounds is not None:
            bounds[gi] = dict(c=[cm[0].bound, cm[1].bound], f=[geo["fields"][k].bound for k in range(4)], rgb=[0.0] * 3,
                              op=0.0)
        if highlight and pv[3] > 0.5:
            assert list(o[8:12]) == [f32(0.3), f32(1.0), f32(0.1), f32(1.0)]
            compared += bbox_decided
            continue
        if sh4.rasterize == "velocity":
            assert o[11] == 0 and list(o[8:11]) == [0, 0, 0] if sc.v < 1e-2 else True, (gi, o)
            compared += bbox_decided
            continue
        op_b = (opac * float(u.global_opacity)).bound
        assert abs(o[11] - col[3]) <= op_b, (gi, o[11], col[3])
        if sh4.rasterize in ("color", "classification"):
            rgb = spherindrical(view.to_abi(), T16, pm[:3], float(f32(f32(u.time) - f32(tt[0]))), duration, shv,
                                int(u.color_space), gpu)
            if sh4.rasterize == "classification" and pv[3] >= 2.0:
                hsv = hsv_e(((E(pv[3]) - 2.0) / float(sh4.num_classes)) * K(6.283185307), E(1.0), E(1.0))
                rgb = [rgb[k] * 0.5 + hsv[k] * 0.5 for k in range(3)]
        elif sh4.rasterize == "position":
            rgb = [(pm[i] - float(u.aabb_min[i])) / (E(float(u.aabb_max[i])) - float(u.aabb_min[i])) for i in range(3)]
        elif sh4.rasterize == "depth":
            cam = [float(x) for x in view.world_position]

            def dist(p3):
                d = [p3[i] - cam[i] for i in range(3)]
                return ((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]).sqrt()
            ends = [dist(mat4_point(T16, [E(float(x)) for x in cloud.position_visibility[int(sorted_ids[i]), :3]])) for i in (n - 1, 1)]
            rgb = depth_rgb_e(dist(pm[:3]), ends[0], ends[1])
        elif sh4.rasterize == "optical_flow":
            rgb = flow_rgb_e(clip16, [float(x) for x in extras.previous_clip_from_world], pm[:3], pw0[:3], float(extras.delta_time))
        for k in range(3):
            assert abs(o[8 + k] - col[k]) <= rgb[k].bound, (gi, sh4.rasterize, k, o[8 + k], col[k], rgb[k].bound)
        if bounds is not None:
            bounds[gi].update(rgb=[rgb[k].bound for k in range(3)], op=op_b)
        compared += bbox_decided
    return compared, undecided, expected


# ---------------------------------------------------------------- whole frames against the emulator
T_STOP = 1.0e-4       # include/bgs.h: a pixel's walk stops once its transmittance falls below 1e-4


def frame_order(cloud, view, u):
    """The walk's order from the keys alone (far -> near, the visible ones), independent of the port's frame."""
    from oracle import oracle as O
    keys = O.keygen(cloud.position_visibility, view.to_abi(), u, 32)
    _, order = O.radix_sort(keys, 32)
    return [int(i) for i in order if keys[i] != 0xFFFFFFFF]


def check_frame(img, cloud, sh4, order, rec, ids, bounds, gpu=False):
    """The port's frame (rgb of img) against the emulator's walk of the same quads, pixel by pixel.

    The walk is render_reference_semantics_4d's -- each quad an affine patch, fs_main per covered pixel centre,
    premultiplied "over" -- taken front to back so that it can apply the port's one documented difference from the
    reference's blend: a pixel stops once its transmittance T < 1e-4.  Nothing else differs, so a pixel's distance
    from the port is bounded by the record errors (`bounds`, from check_records) carried through the blend:

      colour = sum_k w_k c_k, w_k = a_k T_k, T_k = prod_{j<k} (1 - a_j).  sum_i |dw_i / da_k| <= T_k + T_k = 2 T_k
      (the fragment's own weight, and the later weights' sum T_{k+1} / (1 - a_k)), so
      |d colour| <= sum_k T_k (2 |d a_k| C + |d c_k|) + 4u n C,   C = max_k (|c_k| + |d c_k|),

    the last term the f32 blend's own rounding (a product, a sum and the T update per fragment; the kernel's FMAs
    round less).  a_k = min(exp(power) op, 0.999), min 1-Lipschitz:  |d a| <= exp(power) (op expm1(|d power|) +
    |d op|) + 2u a, and on the GPU the blend's exp is ex2.approx of power log2(e): + a (2^-22 + 2u |power|).
    d power comes from the record fields and centre: OBB power = -4.5 (u^2 + v^2), u = ux dx + uy dy (dx = px - cx),
    |d u| <= eb(ux) |dx| + eb(uy) |dy| + (|ux| + |uy|) eb(c) + 2u (|ux dx| + |uy dy|); AABB power =
    -0.5 (c0 mx^2 + c2 my^2) + c1 mx my in half pixels, mx = 2 dx, |d mx| = 2 eb(c).
    Decisions: a pixel centre covered by one side and not the other (|uv| <= 1, within its error of the quad edge) or
    a T crossing 1e-4 within its error make the pixel undecided; the footprint of a splat whose draw decision was
    itself undecided (counted by check_records) is left out.
    -> (compared, undecided, expected, want): `undecided` counts undecided decisions -- an OBB edge pixel, an AABB edge
    (axis-aligned, so a whole row or column of pixel centres shares one margin), a T crossing -- and `expected`
    predicts them the way check_records predicts undecided bboxes: a margin m with error e and per-pixel slope g is
    within e of 0 at a uniformly placed pixel with probability 2e / g.  For an OBB edge, summed over the
    (pixel, fragment) pairs with |m| <= g (about 2 / g of them per unit of edge length), that is sum min(1, e / g);
    each AABB edge is one draw, min(1, 2 e / g)."""
    from wgsl_emu import Vec, ndc_to_pixel
    W, H = img.shape[1], img.shape[0]
    rank = {int(g): r for r, g in enumerate(ids)}
    frags = [[[] for _ in range(W)] for _ in range(H)]        # front-to-back fragments per pixel
    blocked = np.zeros((H, W), bool)
    by_record = np.zeros((H, W), bool)
    amb_edges = set()
    expected = 0.0
    for gi in reversed(order):                               # near -> far
        pv = cloud.position_visibility[gi]
        vs = sh4.vs_points_4d(Vec(pv[0], pv[1], pv[2]), [float(x) for x in cloud.spherindrical_harmonic[gi]],
                              [float(x) for x in cloud.isotropic_rotations[gi]], [float(x) for x in cloud.scale_opacity[gi]],
                              [float(x) for x in cloud.timestamp_timescale[gi]], visibility=float(pv[3]))
        b = bounds.get(gi, "absent")
        if b is None:                                        # an undecided record: its whole footprint is undecided
            o = rec[rank[gi]]
            bb = o[6:8].view(np.uint32)
            x0, x1, y0, y1 = int(bb[0] & 0xFFFF), int(bb[0] >> 16), int(bb[1] & 0xFFFF), int(bb[1] >> 16)
            if x0 <= x1 and y0 <= y1:
                by_record[max(y0 - 1, 0):y1 + 2, max(x0 - 1, 0):x1 + 2] = True
            if vs.get("color") is None:
                continue
        if vs.get("color") is None:
            continue
        P = [ndc_to_pixel(v["position"].xy.v, W, H) for v in vs["vertices"]]
        if b in (None, "absent"):       # drawn here, undecided (or base-culled within its error) in the port
            lo = np.floor(np.min(P, axis=0)).astype(int) - 1
            hi = np.ceil(np.max(P, axis=0)).astype(int) + 1
            by_record[max(lo[1], 0):max(hi[1] + 1, 0), max(lo[0], 0):max(hi[0] + 1, 0)] = True
            continue
        c = ndc_to_pixel(vs["projected_position"].xy.v, W, H)
        A = np.stack([0.5 * (P[2] - P[0]), 0.5 * (P[1] - P[0])], axis=1)
        if not np.all(np.isfinite(A)) or abs(np.linalg.det(A)) < 1e-300:
            continue
        Ai = np.linalg.inv(A)
        lo = np.floor(np.min(P, axis=0)).astype(int) - 2
        hi = np.ceil(np.max(P, axis=0)).astype(int) + 2
        col = vs["color"]
        aabb = sh4.USE_AABB
        Rq = abs(vs["vertices"][3]["bb"].z) if aabb else 0.0
        if aabb:     # each edge is a row or column of pixel centres: one decision, within 2 e / g rows of the lattice
            de = (2 * max(b["c"]) + b["f"][3]) / Rq + 4 * U
            expected += 4 * min(1.0, 2 * de / (2.0 / Rq))
        for y in range(max(lo[1], 0), min(hi[1], H - 1) + 1):
            for x in range(max(lo[0], 0), min(hi[0], W - 1) + 1):
                d = np.array([x + 0.5, y + 0.5]) - c
                uv = Ai @ d
                if aabb:
                    duv = [(2 * b["c"][i] + b["f"][3] * abs(uv[i])) / Rq + 2 * U * (1 + abs(uv[i])) for i in range(2)]
                    g = [2.0 / Rq] * 2
                else:
                    duv = [b["f"][2 * i] * abs(d[0]) + b["f"][2 * i + 1] * abs(d[1]) + (abs(Ai[i, 0]) + abs(Ai[i, 1])) *
                           max(b["c"]) + 2 * U * (abs(Ai[i, 0] * d[0]) + abs(Ai[i, 1] * d[1])) for i in range(2)]
                    g = [math.hypot(Ai[i, 0], Ai[i, 1]) for i in range(2)]
                ambiguous = False
                for i in range(2):      # an edge of the quad: the other coordinate inside it (within its error)
                    m = 1.0 - abs(uv[i])
                    if abs(uv[1 - i]) > 1.0 + duv[1 - i]:
                        continue
                    if abs(m) <= g[i] and not aabb:
                        expected += min(1.0, duv[i] / g[i])
                    if abs(m) <= duv[i]:
                        ambiguous = True
                        amb_edges.add((gi, i, uv[i] > 0) if aabb else (gi, x, y))
                if ambiguous:
                    blocked[y, x] = True
                    continue
                if abs(uv[0]) > 1.0 or abs(uv[1]) > 1.0:
                    continue
                if aabb:
                    mm = Vec(Rq * uv[0], Rq * uv[1])
                    conic = vs["conic"]
                    ddx, ddy = -mm.x, -mm.y
                    power = -0.5 * (conic.x * ddx * ddx + conic.z * ddy * ddy) + conic.y * ddx * ddy
                    dmx = [2 * b["c"][0], 2 * b["c"][1]]
                    dp = (0.5 * (b["f"][0] * ddx * ddx + b["f"][2] * ddy * ddy) + b["f"][1] * abs(ddx * ddy)
                          + (abs(conic.x * ddx) + abs(conic.y * ddy)) * dmx[0] + (abs(conic.z * ddy) + abs(conic.y * ddx)) * dmx[1]
                          + 6 * U * (0.5 * (abs(conic.x) * ddx * ddx + abs(conic.z) * ddy * ddy) + abs(conic.y * ddx * ddy)))
                    if power > 0.0:
                        continue
                else:
                    power = -4.5 * (uv[0] * uv[0] + uv[1] * uv[1])
                    dp = 9.0 * (abs(uv[0]) * duv[0] + abs(uv[1]) * duv[1]) + 3 * U * abs(power)
                ex = math.exp(power)
                a = min(ex * col[3], 0.999)
                da = ex * (col[3] * math.expm1(dp) + b["op"]) + 2 * U * a
                if gpu:
                    da += a * (2.0 ** -22 + 2 * U * abs(power))
                frags[y][x].append((a, da, col.v[:3], b["rgb"]))
    compared = undecided = 0
    want = np.full((H, W, 3), np.nan)          # (NaN: a pixel left out)
    for y in range(H):
        for x in range(W):
            if by_record[y, x]:
                continue
            if blocked[y, x]:
                continue
            T, dT, acc, bound, n = 1.0, 0.0, np.zeros(3), 0.0, 0
            fl = frags[y][x]
            C = max([float(np.max(np.abs(cv) + np.asarray(cb))) for _, _, cv, cb in fl], default=0.0)
            stop_ambiguous = False
            for a, da, cv, cb in fl:
                acc += a * T * np.asarray(cv)
                bound += T * (2 * da * C + max(cb))
                dT = dT * (1 - a) + T * da + 2 * U * T
                Tp, T = T, T * (1 - a)
                n += 1
                if T < T_STOP + dT and Tp >= T_STOP:    # the fragment that crosses 1e-4: T falls across a width Tp a
                    expected += min(1.0, 2 * dT / max(Tp * a, 1e-300))
                if abs(T - T_STOP) <= dT:
                    stop_ambiguous = True
                    break
                if T < T_STOP:
                    break
            if stop_ambiguous:
                undecided += 1
                continue
            bound += 4 * U * n * C + 2.0 ** -40
            want[y, x] = acc
            err = float(np.abs(img[y, x, :3].astype(np.float64) - acc).max())
            assert err <= bound, (x, y, err, bound, len(fl))
            compared += 1
    undecided += len(amb_edges)
    return compared, undecided, expected, want
