"""bgs_cloud_interpolate on the GPU: the blend bit for bit against the CPU oracle (interpolate_oracle/) on every class of
tests/interpolate_cases.py and every layout, at 200 000 gaussians and at 6 M f16 / 2 M f32; both device copies written
(frames of an interpolated cloud are bit-identical to frames of a fresh upload of the oracle's planes); the enqueued
ordering across contexts with no host synchronisation in between; the refusals; and frames of clouds that are never
interpolated keeping their launches."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import interpolate_cases as IC
import particle_cases as PC
from bevy_gaussian_splatting_b200 import abi
from interpolate_oracle import interpolate_oracle as IO
from particle_oracle import particle_oracle as PO
from test_oracle_interpolate import assert_planes

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


@pytest.fixture(scope="module")
def plugin():
    p = B.GaussianSplattingPlugin(0)
    yield p
    p.destroy()


def _ptr(a):
    return np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)


def upload(plugin, layout, planes):
    """A resident cloud holding exactly these upload planes."""
    planes = [np.ascontiguousarray(p) for p in planes]
    n = len(planes[0])
    h = C.c_void_p()
    if layout == "f32":
        st = plugin._lib.bgs_cloud_upload_f32(plugin._ctx, n, *(_ptr(p) for p in planes), C.byref(h))
    else:
        up = plugin._lib.bgs_cloud_upload_f16_cov if layout == "cov" else plugin._lib.bgs_cloud_upload_f16
        st = up(plugin._ctx, n, *(_ptr(p) for p in planes), C.byref(h))
    plugin._check(st)
    return B.PlanarGaussian3dHandle._adopt(plugin, h, n, layout != "f32", layout == "cov")


def clone(plugin, h):
    """The output cloud, made the documented way: an index-mode subset of every gaussian."""
    return plugin.subset(h, np.arange(h.n))


def settings_at(time, time_start=0.0, time_stop=1.0, **kw):
    return B.CloudSettings(time=time, time_start=time_start, time_stop=time_stop, **kw)


def oracle(layout, lhs, rhs, time, time_start=0.0, time_stop=1.0):
    t = IO.factor(time, time_start, time_stop)
    return IO.interpolate(layout, lhs, rhs, t)


def planes_of(cloud: B.PlanarGaussian3d, layout):
    if layout == "f32":
        return (cloud.position_visibility, cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity)
    src = cloud.precomputed_covariance() if layout == "cov" else cloud
    sh, second = src.pack_f16()
    return (cloud.position_visibility, sh, second)


CASES = IC.cases(fill=200_000)


# ---- 1. the blend against the oracle --------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", IC.LAYOUTS)
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_interpolation_matches_oracle(plugin, layout, case):
    lp, rp = case["lhs"][layout], case["rhs"][layout]
    assert len(lp[0]) >= 200_000
    hl = upload(plugin, layout, lp)
    hr = hl if case["same"] else upload(plugin, layout, rp)
    out = clone(plugin, hl)
    try:
        plugin.interpolate(out, hl, hr, settings_at(case["time"], case["time_start"], case["time_stop"]))
        got = plugin.download_planes(out)
        want = oracle(layout, lp, rp, case["time"], case["time_start"], case["time_stop"])
        assert_planes(layout, got, want, case["name"])
        assert_planes(layout, plugin.download_planes(hl), lp, "lhs unchanged")
        assert plugin.sync()
    finally:
        out.destroy(); hr.destroy(); hl.destroy()


@pytest.mark.parametrize("layout,n", [("f16", 6_000_000), ("f32", 2_000_000)])
def test_interpolation_matches_oracle_at_scale(plugin, layout, n):
    lp = planes_of(B.random_gaussians_3d_seeded(n, 1), layout)
    rp = planes_of(B.random_gaussians_3d_seeded(n, 2), layout)
    hl, hr = upload(plugin, layout, lp), upload(plugin, layout, rp)
    out = clone(plugin, hl)
    try:
        for time in (0.37, 1.0):
            plugin.interpolate(out, hl, hr, settings_at(time))
            assert_planes(layout, plugin.download_planes(out), oracle(layout, lp, rp, time), f"{layout} {n} t={time}")
    finally:
        out.destroy(); hr.destroy(); hl.destroy()


# ---- 2. both device copies ------------------------------------------------------------------------------------------
def frame_and_records(plugin, h, settings, view):
    img = plugin.render_view(h, settings, view, fmt="rgba32f")
    rec, ids = plugin.projected()
    return img.copy(), rec.copy(), ids.copy()


SETTINGS_2 = [("3dgs_obb", {}), ("3dgs_aabb", dict(aabb=True)), ("2dgs", dict(gaussian_mode=B.GaussianMode.Gaussian2d)),
              ("selected", dict(draw_mode=B.DrawMode.Selected)),
              ("highlight_selected", dict(draw_mode=B.DrawMode.HighlightSelected)),
              ("depth", dict(rasterize_mode=B.RasterizeMode.Depth)), ("position", dict(rasterize_mode=B.RasterizeMode.Position))]


def small_pair(n, seed):
    lc, rc = B.random_gaussians_3d_seeded(n, seed), B.random_gaussians_3d_seeded(n, seed + 1)
    for c in (lc, rc):
        c.position_visibility[:, :3] *= F(0.1)
    rng = np.random.default_rng(seed)
    lc.position_visibility[:, 3] = rng.uniform(0, 1, n).astype(F)      # visibility crosses 0.5 in the blend
    rc.position_visibility[:, 3] = rng.uniform(0, 1, n).astype(F)
    return lc, rc


@pytest.mark.parametrize("layout", IC.LAYOUTS)
def test_interpolated_frames_equal_fresh_upload(plugin, layout):
    lc, rc = small_pair(30000, 21)
    lp, rp = planes_of(lc, layout), planes_of(rc, layout)
    view = B.headless_view(320, 200)
    hl, hr = upload(plugin, layout, lp), upload(plugin, layout, rp)
    out = clone(plugin, hl)
    try:
        plugin.interpolate(out, hl, hr, settings_at(0.4))
        want_p = oracle(layout, lp, rp, 0.4)
        hf = upload(plugin, layout, want_p)
        hf.aabb = out.aabb = hl.aabb         # the caller's Aabb (the blend does not update it)
        try:
            for name, kw in SETTINGS_2:
                if layout == "cov" and name in ("2dgs", "normal"):
                    continue
                s = B.CloudSettings(global_scale=0.25, binning_rounds=False, **kw)
                got = frame_and_records(plugin, out, s, view)
                want = frame_and_records(plugin, hf, s, view)
                assert len(got[2]) > 100, name
                PC.assert_same(got[0], want[0], f"{name} frame")
                PC.assert_same(got[1], want[1], f"{name} records")
                assert np.array_equal(got[2], want[2]), name
                lf = frame_and_records(plugin, hl, s, view)
                assert not np.array_equal(lf[0], got[0]), name      # the blend changed the frame
        finally:
            hf.destroy()
    finally:
        out.destroy(); hr.destroy(); hl.destroy()


# ---- 3. ordering across contexts, no host synchronisation in between ---------------------------------------------
def reference_frames(ref, layout, states, s, view):
    frames = []
    for planes in states:
        hr = upload(ref, layout, planes)
        try:
            frames.append(ref.render_view(hr, s, view, fmt="rgba32f").copy())
        finally:
            hr.destroy()
    return frames


def test_queued_frames_see_exactly_the_interpolations_enqueued_before_them():
    import torch

    n, w, hgt, layout = 1_000_000, 1920, 1080, "f16"
    lc, rc = B.random_gaussians_3d_seeded(n, 5), B.random_gaussians_3d_seeded(n, 6)
    lp, rp = planes_of(lc, layout), planes_of(rc, layout)
    s = B.CloudSettings(global_scale=0.05, binning_rounds=False)
    view = B.headless_view(w, hgt)
    A, Bp, Cp, ref = (B.GaussianSplattingPlugin(0) for _ in range(4))
    hl, hr = upload(A, layout, lp), upload(A, layout, rp)
    out = clone(A, hl)
    try:
        for p in (A, Bp, Cp):
            p.render_view(out, s, view, to_host=False)
            p.render_view(out, s, view, to_host=False, asynchronous=True)
            assert p.sync()
        outs = [torch.empty((hgt, w, 4), dtype=torch.float32, device="cuda:0") for _ in range(6)]
        torch.cuda.synchronize()
        frame = lambda p, k: p.render_view_to_device(out, s, view, outs[k].data_ptr(), fmt="rgba32f", asynchronous=True)
        frame(A, 0)                                     # S0 = lhs
        Bp.interpolate(out, hl, hr, settings_at(0.25))  # -> S1
        frame(Cp, 1)                                    # S1
        frame(A, 2)                                     # S1
        Cp.interpolate(out, hl, hr, settings_at(0.5))   # -> S2
        frame(Bp, 3)                                    # S2
        A.interpolate(out, hl, hr, settings_at(0.75))   # -> S3
        frame(Cp, 4)                                    # S3
        frame(Bp, 5)                                    # S3
        for p in (A, Bp, Cp):
            assert p.sync()
        got = [o.cpu().numpy() for o in outs]
        states = [lp] + [oracle(layout, lp, rp, t) for t in (0.25, 0.5, 0.75)]
        assert_planes(layout, A.download_planes(out), states[3], "final out")
        want = reference_frames(ref, layout, states, s, view)
        for a in range(4):
            for b in range(a + 1, 4):
                assert not np.array_equal(want[a], want[b])
        for k, state in enumerate((0, 1, 1, 2, 3, 3)):
            assert np.array_equal(got[k].view(np.uint32), want[state].view(np.uint32)), f"frame {k} is not S{state}"
    finally:
        out.destroy(); hr.destroy(); hl.destroy()
        for p in (A, Bp, Cp, ref):
            p.destroy()


def test_writes_of_the_inputs_wait_for_a_queued_interpolation(plugin):
    other = B.GaussianSplattingPlugin(0)
    n, layout = 2_000_000, "f32"
    lc, rc = B.random_gaussians_3d_seeded(n, 8), B.random_gaussians_3d_seeded(n, 9)
    lp, rp = planes_of(lc, layout), planes_of(rc, layout)
    beh = B.random_particle_behaviors(n, 8)
    hl, hr = upload(plugin, layout, lp), upload(plugin, layout, rp)
    o1, o2 = clone(plugin, hl), clone(plugin, hl)
    parts = other.add_particles(beh)
    try:
        plugin.interpolate(o1, hl, hr, settings_at(0.3))            # reads the old inputs
        other.step_particles(hl, parts, 0.5)                        # queued write of lhs on another context
        vis = np.random.default_rng(3).uniform(0, 1, n).astype(F)
        other.set_visibility(hr, vis)                               # synchronous write of rhs on another context
        plugin.interpolate(o2, hl, hr, settings_at(0.3))            # reads the new ones
        want1 = oracle(layout, lp, rp, 0.3)
        new_l = (PO.particle_step(lp[0], beh, 0.5)[0],) + tuple(lp[1:])
        new_r = (np.concatenate([rp[0][:, :3], vis[:, None]], axis=1),) + tuple(rp[1:])
        want2 = oracle(layout, new_l, new_r, 0.3)
        assert_planes(layout, plugin.download_planes(o1), want1, "first out: old inputs")
        assert_planes(layout, plugin.download_planes(o2), want2, "second out: new inputs")
        assert plugin.sync() and other.sync()
    finally:
        parts.destroy(); o1.destroy(); o2.destroy(); hr.destroy(); hl.destroy(); other.destroy()


def test_inputs_destroyed_right_after_the_call(plugin):
    other = B.GaussianSplattingPlugin(0)
    n, layout = 2_000_000, "f16"
    lp = planes_of(B.random_gaussians_3d_seeded(n, 10), layout)
    rp = planes_of(B.random_gaussians_3d_seeded(n, 11), layout)
    hl, hr = upload(other, layout, lp), upload(other, layout, rp)
    out = clone(other, hl)
    try:
        for time in (0.1, 0.2, 0.6):
            plugin.interpolate(out, hl, hr, settings_at(time))
        hl.destroy(); hr.destroy()                   # from the host, with the interpolations still queued on `plugin`
        assert_planes(layout, other.download_planes(out), oracle(layout, lp, rp, 0.6), "out after the inputs are gone")
        assert plugin.sync()
    finally:
        out.destroy(); hr.destroy(); hl.destroy(); other.destroy()


def test_interpolation_sees_particle_steps_queued_on_another_context(plugin):
    other = B.GaussianSplattingPlugin(0)
    n, layout = 1_000_000, "f16"
    lp = planes_of(B.random_gaussians_3d_seeded(n, 12), layout)
    rp = planes_of(B.random_gaussians_3d_seeded(n, 13), layout)
    beh = B.random_particle_behaviors(n, 12)
    hl, hr = upload(plugin, layout, lp), upload(plugin, layout, rp)
    out = clone(plugin, hl)
    parts = other.add_particles(beh)
    try:
        for _ in range(3):
            other.step_particles(hl, parts, 0.25)
            other.step_particles(hr, parts, 0.25)
        plugin.interpolate(out, hl, hr, settings_at(0.5))            # no sync of `other` in between
        pl, b = lp[0], beh
        pr = rp[0]
        for _ in range(3):
            pl, b = PO.particle_step(pl, b, 0.25)
            pr, b = PO.particle_step(pr, b, 0.25)
        want = oracle(layout, (pl,) + tuple(lp[1:]), (pr,) + tuple(rp[1:]), 0.5)
        assert_planes(layout, plugin.download_planes(out), want, "out after queued steps")
        assert plugin.sync() and other.sync()
    finally:
        parts.destroy(); out.destroy(); hr.destroy(); hl.destroy(); other.destroy()


# ---- 4. refusals ----------------------------------------------------------------------------------------------------
def test_refusals_change_nothing(plugin):
    lib, ctx = plugin._lib, plugin._ctx
    lp = planes_of(B.random_gaussians_3d_seeded(1000, 2), "f32")
    rp = planes_of(B.random_gaussians_3d_seeded(1000, 3), "f32")
    hl, hr = upload(plugin, "f32", lp), upload(plugin, "f32", rp)
    out = clone(plugin, hl)
    short = upload(plugin, "f32", tuple(p[:999] for p in rp))
    f16 = upload(plugin, "f16", planes_of(B.random_gaussians_3d_seeded(1000, 3), "f16"))
    cov = upload(plugin, "cov", planes_of(B.random_gaussians_3d_seeded(1000, 3), "cov"))
    f16_out = clone(plugin, f16)
    try:
        before = plugin.download_planes(out)
        before16 = plugin.download_planes(f16_out)
        inf, nan = float("inf"), float("nan")
        calls = [(ctx, out, hl, short), (ctx, out, short, hr), (ctx, out, hl, f16), (ctx, f16_out, f16, cov),
                 (ctx, f16_out, cov, f16), (ctx, out, out, hr), (ctx, out, hl, out)]
        for c, o, l, r in calls:
            assert lib.bgs_cloud_interpolate(c, o._h, l._h, r._h, 0.5, 0.0, 1.0) == abi.BGS_EINVAL
        for args in ((nan, 0, 1), (inf, 0, 1), (0, -inf, 1), (0, 0, nan), (3e38, -3e38, 3e38)):
            assert lib.bgs_cloud_interpolate(ctx, out._h, hl._h, hr._h, *args) == abi.BGS_EINVAL, args
        assert lib.bgs_cloud_interpolate(None, out._h, hl._h, hr._h, 0.5, 0.0, 1.0) == abi.BGS_EINVAL
        assert lib.bgs_cloud_interpolate(ctx, None, hl._h, hr._h, 0.5, 0.0, 1.0) == abi.BGS_EINVAL
        assert lib.bgs_cloud_interpolate(ctx, out._h, None, hr._h, 0.5, 0.0, 1.0) == abi.BGS_EINVAL
        assert lib.bgs_cloud_interpolate(ctx, out._h, hl._h, None, 0.5, 0.0, 1.0) == abi.BGS_EINVAL
        assert plugin.sync()
        assert_planes("f32", plugin.download_planes(out), before, "out after refusals")
        assert_planes("f16", plugin.download_planes(f16_out), before16, "f16 out after refusals")
        # a large finite window is a factor
        plugin.interpolate(out, hl, hr, settings_at(3e38, -3e38, 0.0))
        assert_planes("f32", plugin.download_planes(out), oracle("f32", lp, rp, 3e38, -3e38, 0.0), "t = 1")
    finally:
        for h in (f16_out, cov, f16, short, out, hr, hl):
            h.destroy()


def test_clouds_on_another_device_are_refused():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    p0, p1 = B.GaussianSplattingPlugin(0), B.GaussianSplattingPlugin(1)
    c = B.random_gaussians_3d_seeded(100, 0)
    a0, b0 = p0.add_cloud(c), p0.add_cloud(c)
    a1 = p1.add_cloud(c)
    o0 = clone(p0, a0)
    try:
        before = p0.download_planes(o0)
        for o, l, r in ((o0, a1, b0), (o0, a0, a1), (a1, a0, b0)):
            with pytest.raises(abi.BgsError) as e:
                p0.interpolate(o, l, r, settings_at(0.5))
            assert e.value.status == abi.BGS_EINVAL
        assert_planes("f32", p0.download_planes(o0), before, "out after refusals")
    finally:
        o0.destroy(); a0.destroy(); b0.destroy(); a1.destroy(); p0.destroy(); p1.destroy()


# ---- 5. frames of clouds that are never interpolated ------------------------------------------------------------------
def test_launch_counts_unchanged(plugin):
    view = B.headless_view(320, 200)
    s = B.CloudSettings(global_scale=0.25, binning_rounds=False)
    sd = B.CloudSettings(global_scale=0.25, binning_rounds=False, rasterize_mode=B.RasterizeMode.Depth)
    hl = plugin.add_cloud(B.random_gaussians_3d_seeded(20000, 4))
    hr = plugin.add_cloud(B.random_gaussians_3d_seeded(20000, 5))
    g = plugin.add_cloud(B.random_gaussians_3d_seeded(20000, 6))
    out = clone(plugin, hl)
    try:
        plugin.render_view(g, s, view)
        assert plugin.last_launch_count == 6
        plugin.interpolate(out, hl, hr, settings_at(0.5))
        plugin.render_view(out, s, view)
        assert plugin.last_launch_count == 6           # the blend is not part of the frame
        plugin.render_view(g, s, view)                 # another cloud, never interpolated
        assert plugin.last_launch_count == 6
        plugin.render_view(hl, sd, view)               # an input
        assert plugin.last_launch_count == 7
    finally:
        out.destroy(); hl.destroy(); hr.destroy(); g.destroy()


# ---- 6. the C++ host ------------------------------------------------------------------------------------------------
def test_cpp_host_interpolation_matches_python_host(plugin, tmp_path):
    exe = os.path.join(ROOT, "examples", "headless")
    if not os.path.exists(exe):
        subprocess.run(["make", "-C", os.path.join(ROOT, "examples")], check=True)
    n, w, h, scale, seed, time = 50000, 640, 360, 0.2, 9, "0.35"
    cloud_f, raw_f = str(tmp_path / "cloud.bin"), str(tmp_path / "frame.raw")
    out = subprocess.run([exe, str(n), str(w), str(h), str(scale), str(tmp_path / "0.ppm"), "--dump-cloud", cloud_f, "--raw", raw_f,
                          "--interpolate", str(seed), "--time", time], check=True, capture_output=True, text=True).stdout
    assert "rendered=1" in out and "interpolated:" in out
    buf = np.fromfile(cloud_f, np.uint8)
    f = buf[8:].view(np.float32)
    assert len(f) == 2 * n * 60                      # lhs's planes, then rhs's
    lhs, rhs = (B.PlanarGaussian3d(g[: n * 4].reshape(n, 4), g[n * 4: n * 52].reshape(n, 48), g[n * 52: n * 56].reshape(n, 4),
                                   g[n * 56: n * 60].reshape(n, 4)) for g in (f[: n * 60], f[n * 60:]))
    assert not np.array_equal(lhs.rotation, rhs.rotation)
    hl, hr = plugin.add_cloud(lhs), plugin.add_cloud(rhs)
    o = clone(plugin, hl)
    try:
        plugin.interpolate(o, hl, hr, settings_at(float(time)))
        img = plugin.render_view(o, B.CloudSettings(global_scale=scale), B.headless_view(w, h), fmt="rgba8_srgb")
    finally:
        o.destroy(); hl.destroy(); hr.destroy()
    cpp = np.fromfile(raw_f, np.uint8).reshape(h, w, 4)
    assert np.array_equal(cpp, img)
