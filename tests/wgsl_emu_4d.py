"""The Gaussian4d rule in the WGSL-literal emulator: an INDEPENDENT restatement of the reference's time-conditioned
projection and spherindrical colour, in float64.

TEST INFRASTRUCTURE.  Written from the reference's shaders only (not from temporal_oracle/, csrc/project.cu or
tests/temporal_cases.py), on top of tests/wgsl_emu.py's value semantics and its 3D functions, which it reuses
unchanged: cov2d, get_bounding_box_clip, world_to_clip, in_frustum, world_to_local_direction, srgb_to_linear.

Transliterated (reference file:line):
  outer_product, conditional_cov3d      src/render/gaussian_4d.wgsl:26-130
  spherindrical_harmonics_lookup        src/material/spherindrical_harmonics.wgsl:11-126
  planar4d_color_from_sh                src/render/planar.wgsl:445-452 (convert_sh_color_to_linear: planar.wgsl:91-97)
  vs_points, GAUSSIAN_4D branches       src/render/gaussian.wgsl:185-330, 378-405
  class_to_rgb                          src/material/classification.wgsl (Bevy's hsv_to_rgb)
  calculate_motion_vector, optical_flow_to_rgb   src/material/optical_flow.wgsl

Two places are not float64:
  * `cos` takes the f32 argument WGSL computes, 2.0 * PI * theta rounded at each step from the f32 dir_t and duration,
    and returns math.cos of it.  Near |2 pi theta| = 1e10 one f32 rounding of the argument moves it by ~500 rad, so a
    float64 argument would be a different input, not a more exact one.
  * The atan2 of optical_flow_to_rgb is math.atan2.
Where include/bgs.h (bgs_render_4d, "deliberately differs") departs from the reference, the documented rule is
implemented and marked "bgs.h deviation N".
"""
from __future__ import annotations

import math

import numpy as np

from wgsl_emu import Mat, Shader, Vec, mat3x3, mat4x4, length, normalize, transpose

f32 = np.float32
PI_F32 = float(f32(math.pi))          # const PI = radians(180.0) in f32 (spherindrical_harmonics.wgsl:9)


def outer_product(a, b):
    # gaussian_4d.wgsl:26-35
    return mat3x3(
        a.x * b.x, a.x * b.y, a.x * b.z,
        a.y * b.x, a.y * b.y, a.y * b.z,
        a.z * b.x, a.z * b.y, a.z * b.z,
    )


def hsv_to_rgb(hsv):
    """Bevy's color_operations::hsv_to_rgb: k = (vec3(5, 3, 1) + h / FRAC_PI_3) % 6; v - v s max(0, min(k, min(4 - k, 1)))."""
    h, s, v = hsv
    out = []
    for base in (5.0, 3.0, 1.0):
        x = base + h / (math.pi / 3.0)
        k = x - 6.0 * math.trunc(x / 6.0)           # WGSL float %: x - y * trunc(x / y)
        out.append(v - v * s * max(0.0, min(k, min(4.0 - k, 1.0))))
    return Vec(out)


class Shader4d(Shader):
    """The GAUSSIAN_4D pipeline bound to a view, a cloud uniform, `time` (gaussian_uniforms.time) and the window
    (time_start, time_stop).  OpticalFlow reads `prev_clip_from_world` (a mat4x4) and `delta_time`; Classification
    `num_classes`."""

    def __init__(self, view, gaussian_uniforms, time, time_start, time_stop, use_obb=True, adaptive=True,
                 rasterize="color", prev_clip_from_world=None, delta_time=None, num_classes=1):
        super().__init__(view, gaussian_uniforms, use_obb=use_obb, gaussian_2d=False, adaptive=adaptive, rasterize=rasterize)
        self.time, self.time_start, self.time_stop = float(time), float(time_start), float(time_stop)
        self.prev_clip_from_world = prev_clip_from_world
        self.delta_time = delta_time
        self.num_classes = num_classes

    # gaussian_4d.wgsl:37-130.  rotation, rotation_r: Vec4 as stored (x = w, not normalised); scale: Vec3.
    def conditional_cov3d(self, rotation, rotation_r, scale, timestamp, time_scale, time):
        dt = time - timestamp
        gs = self.gu.global_scale
        S = mat4x4(
            gs * scale.x, 0.0, 0.0, 0.0,
            0.0, gs * scale.y, 0.0, 0.0,
            0.0, 0.0, gs * scale.z, 0.0,
            0.0, 0.0, 0.0, time_scale,
        )
        w = rotation.x; x = rotation.y; y = rotation.z; z = rotation.w
        wr = rotation_r.x; xr = rotation_r.y; yr = rotation_r.z; zr = rotation_r.w
        M_l = mat4x4(
            w, -x, -y, -z,
            x, w, -z, y,
            y, z, w, -x,
            z, -y, x, w,
        )
        M_r = mat4x4(
            wr, -xr, -yr, -zr,
            xr, wr, zr, -yr,
            yr, -zr, wr, xr,
            zr, yr, -xr, wr,
        )
        R = M_r * M_l
        M = R * S
        Sigma = transpose(M) * M
        cov_t = Sigma[3][3]
        with np.errstate(all="ignore"):
            q = np.float64(-0.5) * dt * dt / np.float64(cov_t)      # IEEE: 0 / 0 = NaN, x / 0 = -inf
        marginal_t = math.exp(q) if not math.isnan(q) else math.nan
        mask = marginal_t > 0.05
        out = dict(dt=dt, dir_t=dt, marginal_t=marginal_t, mask=mask, cov_t=cov_t, Sigma=Sigma)
        if not mask:
            out.update(cov3d=[0.0] * 6, delta_mean=Vec(0.0, 0.0, 0.0), opacity_modifier=0.0)
            return out
        cov11 = mat3x3(
            Sigma[0][0], Sigma[0][1], Sigma[0][2],
            Sigma[1][0], Sigma[1][1], Sigma[1][2],
            Sigma[2][0], Sigma[2][1], Sigma[2][2],
        )
        cov12 = Vec(Sigma[0][3], Sigma[1][3], Sigma[2][3])
        cov_op = outer_product(cov12, cov12)
        cov_op_t = mat3x3(
            cov_op[0].x / cov_t, cov_op[0].y / cov_t, cov_op[0].z / cov_t,
            cov_op[1].x / cov_t, cov_op[1].y / cov_t, cov_op[1].z / cov_t,
            cov_op[2].x / cov_t, cov_op[2].y / cov_t, cov_op[2].z / cov_t,
        )
        cov3d_condition = Mat._from_a(cov11._a() - cov_op_t._a())
        delta_mean = (cov12 / cov_t) * dt
        out.update(cov3d=[cov3d_condition[0][0], cov3d_condition[0][1], cov3d_condition[0][2],
                          cov3d_condition[1][1], cov3d_condition[1][2], cov3d_condition[2][2]],
                   delta_mean=delta_mean, opacity_modifier=marginal_t)
        return out

    def time_cos(self, dir_t, k):
        """cos(k * PI * theta), theta = dir_t / duration (spherindrical_harmonics.wgsl:75-78, 102), with WGSL's f32
        argument: every product and quotient rounded to f32 (see the module docstring)."""
        duration = f32(f32(self.time_stop) - f32(self.time_start))
        theta = f32(f32(dir_t) / duration)
        arg = f32(f32(f32(k) * f32(PI_F32)) * theta)
        return math.cos(float(arg)), float(arg)

    # spherindrical_harmonics.wgsl:11-126 at SH_DEGREE 3, SH_DEGREE_TIME 2
    def spherindrical_harmonics_lookup(self, ray_direction, dir_t, sh):
        shc = self.shc
        v3 = lambda i: Vec(sh[i], sh[i + 1], sh[i + 2])  # noqa: E731
        color = Vec(0.5, 0.5, 0.5)
        x = ray_direction.x; y = ray_direction.y; z = ray_direction.z
        l1m1 = shc[1] * y
        l1m0 = shc[2] * z
        l1p1 = shc[3] * x
        xx = x * x; yy = y * y; zz = z * z
        xy = x * y; xz = x * z; yz = y * z
        l2m2 = shc[4] * xy
        l2m1 = shc[5] * yz
        l2m0 = shc[6] * (2.0 * zz - xx - yy)
        l2p1 = shc[7] * xz
        l2p2 = shc[8] * (xx - yy)
        l3m3 = shc[9] * y * (3.0 * xx - yy)
        l3m2 = shc[10] * z * xy
        l3m1 = shc[11] * y * (4.0 * zz - xx - yy)
        l3m0 = shc[12] * z * (2.0 * zz - 3.0 * xx - 3.0 * yy)
        l3p1 = shc[13] * x * (4.0 * zz - xx - yy)
        l3p2 = shc[14] * z * (xx - yy)
        l3p3 = shc[15] * x * (xx - 3.0 * yy)
        l0m0 = shc[0]
        basis = [l0m0, l1m1, l1m0, l1p1, l2m2, l2m1, l2m0, l2p1, l2p2, l3m3, l3m2, l3m1, l3m0, l3p1, l3p2, l3p3]
        for k in range(16):
            color = color + basis[k] * v3(3 * k)
        t1, arg1 = self.time_cos(dir_t, 2.0)
        t2, arg2 = self.time_cos(dir_t, 4.0)
        s1 = Vec(0.0, 0.0, 0.0)
        s2 = Vec(0.0, 0.0, 0.0)
        for k in range(16):
            s1 = s1 + basis[k] * v3(48 + 3 * k)
            s2 = s2 + basis[k] * v3(96 + 3 * k)
        color = color + t1 * s1
        color = color + t2 * s2
        self.last_time_terms = dict(t1=t1, t2=t2, arg1=arg1, arg2=arg2, s1=s1, s2=s2, basis=basis)
        return color

    # planar.wgsl:445-452, 91-97
    def get_color_4d(self, sh, dir_t, ray_direction):
        color = self.spherindrical_harmonics_lookup(ray_direction, dir_t, sh)
        self.last_linear_input = color
        if self.gu.color_space == 1:
            return color
        return self.srgb_to_linear(color)

    def class_to_rgb(self, visualization, sh_color):
        if visualization < 2.0:
            return sh_color
        class_idx = visualization - 2.0
        hue = (class_idx / float(self.num_classes)) * 6.283185307
        hsv = hsv_to_rgb((hue, 1.0, 1.0))
        return sh_color * (1.0 - 0.5) + hsv * 0.5               # mix(a, b, 0.5)

    def optical_flow_rgb(self, world_position, previous_world_position):
        c = self.view.unjittered_clip_from_world * Vec(world_position, 1.0)
        cp = self.prev_clip_from_world * Vec(previous_world_position, 1.0)
        mv = (Vec(c.x, c.y) / c.w - Vec(cp.x, cp.y) / cp.w) * Vec(0.5, -0.5)
        flow = mv / self.delta_time
        radius = length(flow)
        angle = math.atan2(flow.y, flow.x)
        if angle < 0.0:
            angle += 2.0 * math.pi
        m = min(max(radius, 0.0), 1.0)
        return hsv_to_rgb((angle, m, 1.0))

    # gaussian.wgsl:185-436 with GAUSSIAN_4D for one gaussian.  rot8: 8 floats (rotation then rotation_r);
    # tt: (timestamp, time_scale).  Returns None when the quad is discarded, else the varyings and intermediates.
    def vs_points_4d(self, position3, sh, rot8, scale_opacity, tt, visibility=1.0, draw_selected=False,
                     highlight_selected=False):
        gu, view = self.gu, self.view
        position = Vec(position3, 1.0)
        transformed_position = (gu.transform * position).xyz
        previous_transformed_position = transformed_position
        discard_quad = False
        if draw_selected:
            discard_quad = discard_quad or visibility < 0.5
        # bgs.h deviation 1: the base position's frustum test, which the reference applies through the culled key at
        # 32 depth bits (radix.wgsl:86-101 -> gaussian.wgsl:196), at every depth width
        base_clip = self.world_to_clip(transformed_position)
        base_in = self.in_frustum(base_clip.xyz)
        out = dict(base_position=transformed_position, base_clip=base_clip, base_in=base_in, reason=None)
        if not base_in or discard_quad:
            out["reason"] = "base" if not base_in else "selected"
            return out
        opacity = float(scale_opacity[3])
        scale = Vec(scale_opacity[0], scale_opacity[1], scale_opacity[2])
        if self.OPACITY_ADAPTIVE_RADIUS:
            lg = math.log(opacity) if opacity > 0.0 else -math.inf
            cutoff = math.sqrt(max(9.0 + 2.0 * lg, 0.000001))        # from the stored opacity (gaussian.wgsl:229-235)
        else:
            cutoff = 3.0
        g = self.conditional_cov3d(Vec(rot8[0], rot8[1], rot8[2], rot8[3]), Vec(rot8[4], rot8[5], rot8[6], rot8[7]),
                                   scale, float(tt[0]), float(tt[1]), self.time)
        out.update(cutoff=cutoff, cond=g)
        if not g["mask"]:
            out["reason"] = "mask"
            return out
        position_t = Vec(position.xyz + g["delta_mean"], 1.0)
        transformed_position = (gu.transform * position_t).xyz
        projected_position = self.world_to_clip(transformed_position)
        out.update(transformed_position=transformed_position, projected_position=projected_position)
        if not self.in_frustum(projected_position.xyz):
            out["reason"] = "moved"
            return out
        opacity = opacity * g["opacity_modifier"]
        gaussian_cov2d = self.cov2d(transformed_position, g["cov3d"])
        out["cov2d"] = gaussian_cov2d
        quad_vertices = [Vec(-1.0, -1.0), Vec(-1.0, 1.0), Vec(1.0, -1.0), Vec(1.0, 1.0)]
        verts = [(q, self.get_bounding_box_clip(gaussian_cov2d, q, cutoff)) for q in quad_vertices]
        if self.USE_AABB:
            det = gaussian_cov2d.x * gaussian_cov2d.z - gaussian_cov2d.y * gaussian_cov2d.y
            det_inv = 1.0 / det
            out["conic"] = Vec(gaussian_cov2d.z * det_inv, -gaussian_cov2d.y * det_inv, gaussian_cov2d.x * det_inv)
        rgb = Vec(0.0, 0.0, 0.0)
        if self.rasterize in ("color", "classification"):
            ray_direction_world = normalize(transformed_position - view.world_position)
            ray_direction_local = self.world_to_local_direction(ray_direction_world, gu.transform)
            out["ray_direction_local"] = ray_direction_local
            rgb = self.get_color_4d(sh, g["dir_t"], ray_direction_local)
            if self.rasterize == "classification":
                rgb = self.class_to_rgb(visibility, rgb)
        elif self.rasterize == "depth":
            first_position, last_position = self.depth_entries        # sorted entries 1 and count - 1 (base positions)
            min_position = (gu.transform * Vec(last_position, 1.0)).xyz
            max_position = (gu.transform * Vec(first_position, 1.0)).xyz
            camera_position = view.world_position
            rgb = self.depth_to_rgb(length(transformed_position - camera_position),
                                    length(min_position - camera_position), length(max_position - camera_position))
        elif self.rasterize == "optical_flow":
            rgb = self.optical_flow_rgb(transformed_position, previous_transformed_position)   # gaussian.wgsl:201
        elif self.rasterize == "position":
            rgb = (transformed_position - gu.min.xyz) / (gu.max.xyz - gu.min.xyz)
        elif self.rasterize == "velocity":
            time_delta = 1e-3
            fut = self.conditional_cov3d(Vec(rot8[0], rot8[1], rot8[2], rot8[3]), Vec(rot8[4], rot8[5], rot8[6], rot8[7]),
                                         scale, float(tt[0]), float(tt[1]), self.time + time_delta)
            velocity = (fut["delta_mean"] - g["delta_mean"]) / time_delta
            velocity_magnitude = length(velocity)
            scaled_mag = min(max((velocity_magnitude - 1.0) / (2.0 - 1.0), 0.0), 1.0)
            out.update(velocity=velocity, velocity_magnitude=velocity_magnitude, scaled_mag=scaled_mag, future=fut)
            if scaled_mag < 1e-2:
                opacity = 0.0
                rgb = Vec(0.0, 0.0, 0.0)        # bgs.h deviation 2: the reference's normalize(0) * 0 is NaN
            else:
                velocity_normalized = normalize(velocity)
                base_color = 0.5 * (velocity_normalized + Vec(1.0, 1.0, 1.0))
                rgb = base_color * scaled_mag
        color = Vec(rgb, opacity * gu.global_opacity)
        if highlight_selected and visibility > 0.5:
            color = Vec(0.3, 1.0, 0.1, 1.0)
        out["color"] = color
        out["vertices"] = [dict(uv=q, position=Vec(projected_position.xy + bb.xy, projected_position.zw), bb=bb) for q, bb in verts]
        return out


def render_reference_semantics_4d(shader: Shader4d, cloud, order, W, H, draw_selected=False, highlight_selected=False):
    """wgsl_emu.render_reference_semantics for a PlanarGaussian4d: the instanced quads of `order` (far -> near, the
    sorted entry buffer) through vs_points_4d, each an affine patch, fs_main per covered pixel centre, blended
    dst = src + (1 - src.a) dst over a cleared (0, 0, 0, 1) target."""
    from wgsl_emu import ndc_to_pixel
    img = np.zeros((H, W, 4), np.float64)
    img[..., 3] = 1.0
    for gi in order:
        pv = cloud.position_visibility[gi]
        vs = shader.vs_points_4d(Vec(pv[0], pv[1], pv[2]), [float(x) for x in cloud.spherindrical_harmonic[gi]],
                                 [float(x) for x in cloud.isotropic_rotations[gi]], [float(x) for x in cloud.scale_opacity[gi]],
                                 [float(x) for x in cloud.timestamp_timescale[gi]], visibility=float(pv[3]),
                                 draw_selected=draw_selected, highlight_selected=highlight_selected)
        if vs.get("color") is None:
            continue
        P = [ndc_to_pixel(v["position"].xy.v, W, H) for v in vs["vertices"]]
        c = 0.25 * (P[0] + P[1] + P[2] + P[3])
        A = np.stack([0.5 * (P[2] - P[0]), 0.5 * (P[1] - P[0])], axis=1)
        if not np.all(np.isfinite(A)) or abs(np.linalg.det(A)) < 1e-300:
            continue
        Ainv = np.linalg.inv(A)
        lo = np.floor(np.min(P, axis=0)).astype(int) - 1
        hi = np.ceil(np.max(P, axis=0)).astype(int) + 1
        mm_corner = [v["bb"].zw for v in vs["vertices"]]
        for y in range(max(lo[1], 0), min(hi[1], H - 1) + 1):
            for x in range(max(lo[0], 0), min(hi[0], W - 1) + 1):
                uv = Ainv @ (np.array([x + 0.5, y + 0.5]) - c)
                if abs(uv[0]) > 1.0 or abs(uv[1]) > 1.0:
                    continue
                mm = Vec(mm_corner[3].x * uv[0], mm_corner[3].y * uv[1]) if shader.USE_AABB else None
                src = shader.fs_main(vs, Vec(uv[0], uv[1]), mm)
                if src is None:
                    continue
                img[y, x] = src.v + (1.0 - src.v[3]) * img[y, x]
    return img
