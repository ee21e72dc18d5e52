"""RasterizeMode::Classification and RasterizeMode::OpticalFlow: an independent numpy f32 restatement of their colour
sources (include/bgs.h, "The rule, exactly": gaussian.wgsl:312-421, material/classification.wgsl:9-27,
material/optical_flow.wgsl:16-53, Bevy's hsv_to_rgb), the inputs built to reach each of their branches, and the scenes
the GPU tests render.

Every f32 operation is one numpy float32 operation (correctly rounded, no contraction), in the order the rule writes.
atan2 is the policy's fixed f64 series, restated here in numpy float64 operations."""
from __future__ import annotations

import numpy as np

f32 = np.float32
FRAC_PI_3 = f32(1.0471975512)          # bevy_render::maths, rounded to f32
PI_2 = f32(6.28318530718)
TAU_CLASS = f32(6.283185307)           # classification.wgsl's literal
NUM_CLASSES = (1, 3, 1 << 20)


def hsv_to_rgb(h, s, v):
    """k = (vec3(5, 3, 1) + h / FRAC_PI_3) % 6 (WGSL f32 %: x - y * trunc(x / y)); v - v s max(0, min(k, min(4 - k, 1)))."""
    h, s, v = (np.asarray(a, f32) for a in np.broadcast_arrays(h, s, v))
    out = []
    with np.errstate(invalid="ignore", over="ignore"):
        hk = h / FRAC_PI_3
        vs = v * s
        for base in (f32(5), f32(3), f32(1)):
            x = base + hk
            k = x - f32(6) * np.trunc(x / f32(6))
            out.append(v - vs * np.fmax(f32(0), np.fmin(k, np.fmin(f32(4) - k, f32(1)))))
    return np.stack(out, -1).astype(f32)


def atan2(y, x):
    """The fixed-series atan2 of the FP policy, in float64 steps, rounded to f32."""
    y, x = np.asarray(y, f32), np.asarray(x, f32)
    with np.errstate(all="ignore"):
        ay, ax = np.abs(y.astype(np.float64)), np.abs(x.astype(np.float64))
        steep = ay > ax
        t = np.where(ax == ay, np.where(ax == 0.0, 0.0, 1.0), np.where(steep, ax / ay, ay / ax))
        hi = t > 0.41421356237309503
        base = np.where(hi, 0.7853981633974483, 0.0)
        u = np.where(hi, (t - 1.0) / (t + 1.0), t)
        z = u * u
        p = np.full_like(z, -1.0 / 43.0)
        for k in range(20, -1, -1):
            p = p * z + (-1.0 if k & 1 else 1.0) / float(2 * k + 1)
        r = base + u * p
        r = np.where(steep, 1.5707963267948966 - r, r)
        r = np.where(np.signbit(x), 3.141592653589793 - r, r)
        r = np.where(np.signbit(y), -r, r)
        r = np.where(np.isnan(x) | np.isnan(y), np.nan, r)
    return r.astype(f32)


def class_colour(sh_rgb, vis, num_classes: int):
    """vis < 2: sh.  Else mix(sh, hsv_to_rgb(((vis - 2) / f32(num_classes)) * 6.283185307, 1, 1), 0.5)."""
    sh = np.asarray(sh_rgb, f32).reshape(-1, 3)
    vis = np.asarray(vis, f32).ravel()
    with np.errstate(invalid="ignore", over="ignore"):
        hue = ((vis - f32(2)) / f32(num_classes)) * TAU_CLASS
        hsv = hsv_to_rgb(hue, f32(1), f32(1))
        mixed = sh * (f32(1) - f32(0.5)) + hsv * f32(0.5)
    return np.where((vis < f32(2))[:, None], sh, mixed).astype(f32)


def mat4_point(m, p):
    """M (p, 1) with m 16 floats column-major, summed ((m0 x + m1 y) + m2 z) + m3 per row; p (n, 3) -> (n, 4)."""
    m = np.asarray(m, f32).reshape(4, 4).T          # row-major
    p = np.asarray(p, f32)
    return np.stack([((m[r, 0] * p[:, 0] + m[r, 1] * p[:, 1]) + m[r, 2] * p[:, 2]) + m[r, 3] for r in range(4)], 1)


def flow_colour(pos_vis, transform, clip, prev_clip, delta_time):
    """p = transform (pos, 1); mv = (c.xy / c.w - c'.xy / c'.w) (0.5, -0.5); flow = mv / dt; rgb = hsv_to_rgb(atan2
    (+ PI_2 below 0), clamp(length(flow), 0, 1), 1)."""
    pos = np.asarray(pos_vis, f32).reshape(-1, 4)
    dt = f32(delta_time)
    with np.errstate(all="ignore"):
        pw = mat4_point(transform, pos[:, :3])
        c, cp = mat4_point(clip, pw[:, :3]), mat4_point(prev_clip, pw[:, :3])
        mvx = (c[:, 0] / c[:, 3] - cp[:, 0] / cp[:, 3]) * f32(0.5)
        mvy = (c[:, 1] / c[:, 3] - cp[:, 1] / cp[:, 3]) * f32(-0.5)
        fx, fy = mvx / dt, mvy / dt
        radius = np.sqrt(fx * fx + fy * fy)
        angle = atan2(fy, fx)
        angle = np.where(angle < f32(0), angle + PI_2, angle).astype(f32)
        return hsv_to_rgb(angle, np.fmin(np.fmax(radius, f32(0)), f32(1)), f32(1))


def same_bits(a, b):
    """Bit for bit, with any NaN equal to any NaN (NaN payloads are not part of the policy)."""
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


# ---------------------------------------------------------------------------------------------------------------------
# inputs that reach each branch

def class_labels(num_classes: int):
    """vis below 2, exactly 2, each class boundary 2 + k (and one ulp either side), fractional labels, 2 + num_classes and
    beyond (the hue wraps), huge labels (2 + k num_classes for k of 6e6 .. 1e12, where h / FRAC_PI_3 passes 2^24 and WGSL's
    x - 6 trunc(x / 6) is no longer fmodf's exact remainder), NaN and +-inf."""
    n = num_classes
    ks = np.unique(np.array([0, 1, 2, n // 2, n - 1, n, n + 1, 2 * n, 3 * n + 1], np.float64))
    b = (f32(2) + ks.astype(f32)).astype(f32)
    v = [np.array([-np.inf, -1.0, 0.0, 0.5, 1.0, 1.5, np.nextafter(f32(2), f32(0)), 2.0], f32), b,
         np.nextafter(b, f32(np.inf)), np.nextafter(b, f32(-np.inf)), b + f32(0.25), b + f32(0.5),
         (f32(2) + (np.array([6e6 + 1, 1.7e7 + 3, 1e12 + 5]) * n).astype(f32)).astype(f32),
         np.array([1e30, np.nan, np.inf, -np.nan], f32)]
    return np.concatenate(v).astype(f32)


def sextant_flows():
    """(fx, fy) in each of the six hue sextants, both below and above radius 1, the exact axes (+-0 and +-pi), zero."""
    out = []
    for i in range(6):
        th = (i + 0.5) * np.pi / 3
        for r in (0.25, 0.999, 1.0, 3.0):
            out.append((r * np.cos(th), r * np.sin(th)))
    out += [(0.5, 0.0), (0.5, -0.0), (-0.5, 0.0), (-0.5, -0.0), (0.0, 0.5), (0.0, -0.5), (0.0, 0.0), (-0.0, 0.0),
            (0.0, -0.0), (-0.0, -0.0), (2.0, 0.0), (-2.0, -0.0), (np.inf, 1.0), (-np.inf, 1.0), (1.0, np.inf),
            (np.inf, np.inf), (-np.inf, -np.inf), (np.nan, 1.0), (1e-40, 1e-40), (1e-30, -3e-30)]
    return np.array(out, f32)


def translated(fx: float, fy: float):
    """previous_clip_from_world = the identity moved by (-2 fx, 2 fy): with clip_from_world = the identity and dt = 1, a
    point at the origin moves by flow (fx, fy) exactly (0 - t is exact, and so are * 0.5 and / 1)."""
    m = np.eye(4, dtype=f32)
    m[0, 3], m[1, 3] = f32(-2.0) * f32(fx), f32(2.0) * f32(fy)
    return np.ascontiguousarray(m.T).reshape(-1)


def camera_matrices(seed: int = 0):
    """clip_from_world pairs (current, previous): a perspective camera, then moved by a small, large and zero step,
    rotated, and one whose previous w is <= 0 for part of the scene."""
    rng = np.random.default_rng(seed)

    def persp(fov, aspect, near, eye, yaw):
        f = 1.0 / np.tan(fov / 2)
        P = np.array([[f / aspect, 0, 0, 0], [0, f, 0, 0], [0, 0, 0, near], [0, 0, -1, 0]], np.float64)   # reverse-z
        c, s = np.cos(yaw), np.sin(yaw)
        R = np.array([[c, 0, -s, 0], [0, 1, 0, 0], [s, 0, c, 0], [0, 0, 0, 1]], np.float64)
        T = np.eye(4)
        T[:3, 3] = -np.asarray(eye, np.float64)
        return (P @ R @ T).astype(f32)

    cur = persp(0.9, 1.5, 0.1, (0, 0, 5), 0.0)
    prevs = {"step": persp(0.9, 1.5, 0.1, (0.02, 0.01, 5), 0.0), "jump": persp(0.9, 1.5, 0.1, (1.5, -0.7, 4.0), 0.3),
             "still": cur.copy(), "yaw": persp(0.9, 1.5, 0.1, (0, 0, 5), 0.05),
             "behind": persp(0.9, 1.5, 0.1, (0, 0, -2.0), 0.0)}
    col = lambda m: np.ascontiguousarray(m.T).reshape(-1)   # noqa: E731  row-major -> column-major
    return col(cur), {k: col(v) for k, v in prevs.items()}, rng
