"""bgs_cloud_particles_step on the GPU: the step bit for bit against the CPU oracle (particle_oracle/) on every class of
tests/particle_cases.py and every layout; both device copies of the position moved (frames of a stepped cloud are
bit-identical to frames of a fresh upload of the oracle's positions); the enqueued ordering across contexts with no
host synchronisation in between; the steps against the synchronous writers; the refusals; and frames of clouds that
are never stepped keeping their launches."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import particle_cases as PC
from bevy_gaussian_splatting_b200 import abi
from particle_oracle import particle_oracle as PO
from select_oracle import select_oracle as SO

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def plugin():
    p = B.GaussianSplattingPlugin(0)
    yield p
    p.destroy()


def host_cloud(pos: np.ndarray, seed: int = 0) -> B.PlanarGaussian3d:
    c = B.random_gaussians_3d_seeded(len(pos), seed)
    c.position_visibility[:] = pos
    return c


def add(plugin, cloud, layout):
    return plugin.add_cloud(cloud, f16=layout == "f16", precompute_covariance=layout == "cov")


def step_and_check(plugin, h, case):
    """Every dt of the case as one step each, then positions and behaviours against the oracle."""
    parts = plugin.add_particles(case["behaviors"])
    try:
        for dt in case["dts"]:
            plugin.step_particles(h, parts, dt)
        want_p, want_b = PO.particle_steps(case["pos"], case["behaviors"], case["dts"])
        PC.assert_same(plugin.positions(h), want_p, f"{case['name']} positions")
        PC.assert_same_behaviors(parts.get(), want_b, case["name"])
        assert plugin.sync()
        return want_p, want_b
    finally:
        parts.destroy()


CASES = PC.cases(scale=40)          # bulk classes at 200 000 gaussians, many_steps at 80 000


# ---- 1. the step against the oracle -------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["f32", "f16", "cov"])
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_steps_match_oracle(plugin, layout, case):
    assert any(len(c["pos"]) == 200_000 for c in CASES)
    h = add(plugin, host_cloud(case["pos"], len(case["pos"]) % 7), layout)
    try:
        step_and_check(plugin, h, case)
    finally:
        h.destroy()


def test_steps_match_oracle_at_six_million_f16(plugin):
    n = 6_000_000
    cloud = B.random_gaussians_3d_seeded(n, 0)
    beh = B.random_particle_behaviors(n, 0)
    h = plugin.add_cloud(cloud, f16=True)
    try:
        step_and_check(plugin, h, {"name": "c3", "pos": cloud.position_visibility, "behaviors": beh, "dts": [1 / 60, 1 / 144]})
    finally:
        h.destroy()


# ---- 2. both device copies ----------------------------------------------------------------------------------------
def frame_and_records(plugin, h, settings, view):
    img = plugin.render_view(h, settings, view, fmt="rgba32f")
    rec, ids = plugin.projected()
    return img.copy(), rec.copy(), ids.copy()


SETTINGS_2 = [("3dgs_obb", {}), ("3dgs_aabb", dict(aabb=True)), ("2dgs", dict(gaussian_mode=B.GaussianMode.Gaussian2d)),
              ("selected", dict(draw_mode=B.DrawMode.Selected)),
              ("highlight_selected", dict(draw_mode=B.DrawMode.HighlightSelected)),
              ("depth", dict(rasterize_mode=B.RasterizeMode.Depth)), ("position", dict(rasterize_mode=B.RasterizeMode.Position))]


@pytest.mark.parametrize("layout", ["f32", "f16", "cov"])
def test_stepped_frames_equal_fresh_upload(plugin, layout):
    case = PC.w_crossing(30000, 21)
    cloud = host_cloud(case["pos"], 21)
    cloud.position_visibility[:, :3] *= np.float32(0.1)
    case["pos"] = cloud.position_visibility.copy()
    view = B.headless_view(320, 200)
    h = add(plugin, cloud, layout)
    parts = plugin.add_particles(case["behaviors"])
    try:
        for dt in case["dts"]:
            plugin.step_particles(h, parts, dt)
        want_p, _ = PO.particle_steps(case["pos"], case["behaviors"], case["dts"])
        PC.assert_same(plugin.positions(h), want_p, "positions")
        w0, w1 = case["pos"][:, 3], want_p[:, 3]
        assert ((w0 < 0.5) & (w1 >= 0.5)).any() and ((w0 >= 0.5) & (w1 < 0.5)).any()
        fresh = host_cloud(want_p, 21)
        fresh.spherical_harmonic[:], fresh.rotation[:], fresh.scale_opacity[:] = \
            cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity
        hf = add(plugin, fresh, layout)
        hf.aabb = h.aabb             # the caller's Aabb (the step does not update it; RasterizeMode::Position reads it)
        try:
            for name, kw in SETTINGS_2:
                if layout == "cov" and name == "2dgs":
                    continue
                s = B.CloudSettings(global_scale=0.25, binning_rounds=False, **kw)
                got = frame_and_records(plugin, h, s, view)
                want = frame_and_records(plugin, hf, s, view)
                assert len(got[2]) > 100, name
                PC.assert_same(got[0], want[0], f"{name} frame")
                PC.assert_same(got[1], want[1], f"{name} records")
                assert np.array_equal(got[2], want[2]), name
        finally:
            hf.destroy()
    finally:
        parts.destroy()
        h.destroy()


# ---- 3. ordering across contexts, no host synchronisation in between --------------------------------------------
def test_queued_frames_see_exactly_the_steps_enqueued_before_them():
    import torch

    n, w, hgt = 1_000_000, 1920, 1080
    cloud = B.random_gaussians_3d_seeded(n, 5)
    beh = B.random_particle_behaviors(n, 5)
    beh2 = B.random_particle_behaviors(n // 4, 6)
    beh2["indices"][:, 0] = np.random.default_rng(6).choice(n, n // 4, replace=False).astype(np.uint32)
    s = B.CloudSettings(global_scale=0.05, binning_rounds=False)
    view = B.headless_view(w, hgt)
    A, Bp, Cp, ref = (B.GaussianSplattingPlugin(0) for _ in range(4))
    h = A.add_cloud(cloud, f16=True)
    pa = A.add_particles(beh)
    pb = Bp.add_particles(beh2)
    dt1, dt2, dt3 = 1 / 60, 1 / 144, 0.5
    try:
        # warm every context's pair buffer (and its queued-frame path) on this cloud and view
        for p in (A, Bp, Cp):
            p.render_view(h, s, view, to_host=False)
            p.render_view(h, s, view, to_host=False, asynchronous=True)
            assert p.sync()
        outs = [torch.empty((hgt, w, 4), dtype=torch.float32, device="cuda:0") for _ in range(6)]
        torch.cuda.synchronize()
        frame = lambda p, k: p.render_view_to_device(h, s, view, outs[k].data_ptr(), fmt="rgba32f", asynchronous=True)
        frame(A, 0)                  # P0
        Bp.step_particles(h, pa, dt1)   # -> P1 (queued on B after A's frame)
        frame(Cp, 1)                 # P1
        frame(A, 2)                  # P1
        Cp.step_particles(h, pb, dt2)   # -> P2 (another behaviours object)
        frame(Bp, 3)                 # P2
        A.step_particles(h, pa, dt3)    # -> P3 (pa again, now from A: after B's step of it)
        frame(Cp, 4)                 # P3
        frame(Bp, 5)                 # P3
        for p in (A, Bp, Cp):
            assert p.sync()
        got = [o.cpu().numpy() for o in outs]

        p0 = cloud.position_visibility
        p1, b1 = PO.particle_step(p0, beh, dt1)
        p2, _ = PO.particle_step(p1, beh2, dt2)
        p3, b3 = PO.particle_step(p2, b1, dt3)
        PC.assert_same(A.positions(h), p3, "final positions")
        PC.assert_same_behaviors(pa.get(), b3, "final behaviours")
        want = []
        for pos in (p0, p1, p2, p3):
            c = B.PlanarGaussian3d(pos, cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity)
            hr = ref.add_cloud(c, f16=True)
            try:
                want.append(ref.render_view(hr, s, view, fmt="rgba32f").copy())
            finally:
                hr.destroy()
        for a in range(4):
            for b in range(a + 1, 4):
                assert not np.array_equal(want[a], want[b])      # every step changes the frame
        for k, state in enumerate((0, 1, 1, 2, 3, 3)):
            assert np.array_equal(got[k].view(np.uint32), want[state].view(np.uint32)), f"frame {k} is not P{state}"
    finally:
        pa.destroy(); pb.destroy(); h.destroy()
        for p in (A, Bp, Cp, ref):
            p.destroy()


# ---- 4. steps against the synchronous writers ---------------------------------------------------------------------
def cube(lo, hi):
    v = np.array([[x, y, z] for x in (lo, hi) for y in (lo, hi) for z in (lo, hi)], np.float32)
    f = [(0, 1, 3), (0, 3, 2), (4, 6, 7), (4, 7, 5), (0, 4, 5), (0, 5, 1), (2, 3, 7), (2, 7, 6), (0, 2, 6), (0, 6, 4),
         (1, 5, 7), (1, 7, 3)]
    return v, np.array(f, np.uint32)


def test_selections_on_another_context_see_queued_steps(plugin):
    other = B.GaussianSplattingPlugin(0)
    cloud = B.random_gaussians_3d_seeded(400_000, 7)
    cloud.position_visibility[:, :3] *= np.float32(0.05)
    beh = B.random_particle_behaviors(len(cloud), 7)
    h = plugin.add_cloud(cloud)
    parts = plugin.add_particles(beh)
    try:
        pos = cloud.position_visibility
        for k in range(3):
            plugin.step_particles(h, parts, 0.25)
            pos, beh = PO.particle_step(pos, beh, 0.25)
        sel = other.select_sparse(h, B.SparseSelect(0.02, 3))       # queued steps on `plugin`, not synced
        mask, count = SO.select_sparse(pos, 0.02, 3, grid=True)
        assert sel == count and np.array_equal(other.visibility(h), mask.astype(np.float32))
        pos[:, 3] = mask.astype(np.float32)
        plugin.step_particles(h, parts, 0.1)
        pos, beh = PO.particle_step(pos, beh, 0.1)
        v, i = cube(-0.5, 0.5)
        inside = other.select_in_mesh(h, v, i)
        m2, c2 = SO.select_in_mesh(pos, v, i)
        assert inside == c2 and 0 < c2 < len(pos)
        assert np.array_equal(other.visibility(h), m2.astype(np.float32))
        pos[:, 3] = m2.astype(np.float32)
        # visibility_set on one context, then a step on the other moves the set values
        vis = np.random.default_rng(1).uniform(0, 1, len(pos)).astype(np.float32)
        other.set_visibility(h, vis)
        pos[:, 3] = vis
        plugin.step_particles(h, parts, 1 / 60)
        pos, beh = PO.particle_step(pos, beh, 1 / 60)
        PC.assert_same(other.positions(h), pos, "positions after set_visibility + step")
        PC.assert_same(other.visibility(h), pos[:, 3], "visibility after step")
        PC.assert_same_behaviors(parts.get(), beh, "behaviours")
        assert plugin.sync()
    finally:
        parts.destroy(); h.destroy(); other.destroy()


@pytest.mark.parametrize("what", ["cloud", "particles"])
def test_destroy_with_steps_queued_on_another_context(plugin, what):
    other = B.GaussianSplattingPlugin(0)
    n = 2_000_000
    h = other.add_cloud(B.random_gaussians_3d_seeded(n, 3), f16=True)
    parts = other.add_particles(B.random_particle_behaviors(n, 3))
    try:
        for _ in range(8):
            plugin.step_particles(h, parts, 1 / 60)
        if what == "cloud":
            h.destroy()
        else:
            parts.destroy()
        assert plugin.sync()
    finally:
        parts.destroy(); h.destroy(); other.destroy()


# ---- 5. refusals --------------------------------------------------------------------------------------------------
def test_refusals_change_nothing(plugin):
    lib, ctx = plugin._lib, plugin._ctx
    cloud = B.random_gaussians_3d_seeded(1000, 2)
    h = plugin.add_cloud(cloud)
    beh = B.random_particle_behaviors(1000, 2)
    parts = plugin.add_particles(beh)
    try:
        pos0, b0 = plugin.positions(h), parts.get()

        def einval(call):
            with pytest.raises(abi.BgsError) as e:
                call()
            assert e.value.status == abi.BGS_EINVAL

        dup = beh.copy()
        dup["indices"][5, 0] = 4
        einval(lambda: plugin.add_particles(dup))
        dup["indices"][5, 0] = 0x80000000                  # inactive: fine
        plugin.add_particles(dup).destroy()
        einval(lambda: plugin.add_particles(B.ParticleBehaviors(0)))
        for dt in (float("nan"), float("inf"), float("-inf")):
            einval(lambda: plugin.step_particles(h, parts, dt))
        big = B.random_particle_behaviors(1001, 2)          # names gaussian 1000 of a 1000-gaussian cloud
        pbig = plugin.add_particles(big)
        try:
            einval(lambda: plugin.step_particles(h, pbig, 1 / 60))
            PC.assert_same_behaviors(pbig.get(), big, "refused behaviours")
        finally:
            pbig.destroy()
        p = C.c_void_p()
        bp = beh.ctypes.data_as(C.c_void_p)
        buf = np.empty((1000, 4), np.float32)
        assert lib.bgs_particles_create(None, bp, 1000, C.byref(p)) == abi.BGS_EINVAL
        assert lib.bgs_particles_create(ctx, None, 1000, C.byref(p)) == abi.BGS_EINVAL
        assert lib.bgs_particles_create(ctx, bp, 1000, None) == abi.BGS_EINVAL
        assert lib.bgs_particles_create(ctx, bp, 1 << 30, C.byref(p)) == abi.BGS_EINVAL
        assert lib.bgs_particles_get(None, parts._h, buf.ctypes.data_as(C.c_void_p)) == abi.BGS_EINVAL
        assert lib.bgs_particles_get(ctx, None, buf.ctypes.data_as(C.c_void_p)) == abi.BGS_EINVAL
        assert lib.bgs_particles_get(ctx, parts._h, None) == abi.BGS_EINVAL
        assert lib.bgs_cloud_particles_step(None, h._h, parts._h, 0.1) == abi.BGS_EINVAL
        assert lib.bgs_cloud_particles_step(ctx, None, parts._h, 0.1) == abi.BGS_EINVAL
        assert lib.bgs_cloud_particles_step(ctx, h._h, None, 0.1) == abi.BGS_EINVAL
        assert lib.bgs_cloud_positions_get(None, h._h, buf.ctypes.data_as(C.c_void_p)) == abi.BGS_EINVAL
        assert lib.bgs_cloud_positions_get(ctx, None, buf.ctypes.data_as(C.c_void_p)) == abi.BGS_EINVAL
        assert lib.bgs_cloud_positions_get(ctx, h._h, None) == abi.BGS_EINVAL
        lib.bgs_particles_destroy(None)
        assert np.array_equal(plugin.positions(h).view(np.uint32), pos0.view(np.uint32))
        PC.assert_same_behaviors(parts.get(), b0, "behaviours after refusals")
        assert np.array_equal(pos0, cloud.position_visibility)
        # zero and negative dt are legal
        plugin.step_particles(h, parts, 0.0)
        plugin.step_particles(h, parts, -1 / 60)
        want, _ = PO.particle_steps(cloud.position_visibility, beh, [0.0, -1 / 60])
        PC.assert_same(plugin.positions(h), want, "dt 0 and -1/60")
    finally:
        parts.destroy(); h.destroy()


def test_particles_on_another_device_are_refused():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    p0, p1 = B.GaussianSplattingPlugin(0), B.GaussianSplattingPlugin(1)
    h0 = p0.add_cloud(B.random_gaussians_3d_seeded(100, 0))
    h1 = p1.add_cloud(B.random_gaussians_3d_seeded(100, 0))
    q0 = p0.add_particles(B.random_particle_behaviors(100, 0))
    q1 = p1.add_particles(B.random_particle_behaviors(100, 0))
    out = np.empty(100, B.PARTICLE_BEHAVIOR_DTYPE)
    try:
        for call in (lambda: p0.step_particles(h1, q0, 0.1), lambda: p0.step_particles(h0, q1, 0.1), lambda: p0.positions(h1),
                     lambda: p0._check(p0._lib.bgs_particles_get(p0._ctx, q1._h, out.ctypes.data_as(C.c_void_p)))):
            with pytest.raises(abi.BgsError) as e:
                call()
            assert e.value.status == abi.BGS_EINVAL
    finally:
        q0.destroy(); q1.destroy(); h0.destroy(); h1.destroy(); p0.destroy(); p1.destroy()


# ---- 6. frames of clouds that are never stepped -------------------------------------------------------------------
def test_launch_counts_unchanged(plugin):
    view = B.headless_view(320, 200)
    s = B.CloudSettings(global_scale=0.25, binning_rounds=False)
    sd = B.CloudSettings(global_scale=0.25, binning_rounds=False, rasterize_mode=B.RasterizeMode.Depth)
    h = plugin.add_cloud(B.random_gaussians_3d_seeded(20000, 4))
    g = plugin.add_cloud(B.random_gaussians_3d_seeded(20000, 5))
    parts = plugin.add_particles(B.random_particle_behaviors(20000, 4))
    try:
        plugin.render_view(h, s, view)
        assert plugin.last_launch_count == 6           # key-gen, depth sort, projection, binning, tile sort, blend
        plugin.render_view(h, sd, view)
        assert plugin.last_launch_count == 7           # + the depth range
        plugin.step_particles(h, parts, 1 / 60)
        plugin.render_view(h, s, view)
        assert plugin.last_launch_count == 6           # the step is not part of the frame
        plugin.render_view(g, s, view)                 # another cloud, never stepped
        assert plugin.last_launch_count == 6
        plugin.render_view(h, sd, view)
        assert plugin.last_launch_count == 7
    finally:
        parts.destroy(); h.destroy(); g.destroy()


# ---- 7. the C++ host ------------------------------------------------------------------------------------------------
def test_cpp_host_particles_match_python_host(plugin, tmp_path):
    exe = os.path.join(ROOT, "examples", "headless")
    if not os.path.exists(exe):
        subprocess.run(["make", "-C", os.path.join(ROOT, "examples")], check=True)
    n, w, h, scale, np_, k, dt = 50000, 640, 360, 0.2, 30000, 5, "0.0125"
    cloud_f, raw_f, part_f = str(tmp_path / "cloud.bin"), str(tmp_path / "frame.raw"), str(tmp_path / "particles.bin")
    out = subprocess.run([exe, str(n), str(w), str(h), str(scale), str(tmp_path / "0.ppm"), "--dump-cloud", cloud_f, "--raw", raw_f,
                          "--particles", str(np_), "--steps", str(k), "--dt", dt, "--dump-particles", part_f],
                         check=True, capture_output=True, text=True).stdout
    assert "rendered=1" in out and "particles:" in out
    buf = np.fromfile(cloud_f, np.uint8)
    f = buf[8:].view(np.float32)
    cloud = B.PlanarGaussian3d(f[: n * 4].reshape(n, 4), f[n * 4: n * 52].reshape(n, 48), f[n * 52: n * 56].reshape(n, 4),
                               f[n * 56: n * 60].reshape(n, 4))
    pb = np.fromfile(part_f, np.uint8)
    assert int(pb[:8].view(np.uint64)[0]) == np_
    before = pb[8: 8 + np_ * 64].view(B.PARTICLE_BEHAVIOR_DTYPE)
    after = pb[8 + np_ * 64: 8 + 2 * np_ * 64].view(B.PARTICLE_BEHAVIOR_DTYPE)
    moved = pb[8 + 2 * np_ * 64:].view(np.float32).reshape(n, 4)
    assert np.array_equal(before["indices"][:, 0], np.arange(np_))
    assert np.abs(before["velocity"]).max() < 1 and np.abs(before["jerk"]).max() < 1e-4
    hnd = plugin.add_cloud(cloud)
    parts = plugin.add_particles(before)
    try:
        for _ in range(k):
            plugin.step_particles(hnd, parts, float(dt))
        PC.assert_same(plugin.positions(hnd), moved, "C++ host positions")
        PC.assert_same_behaviors(parts.get(), after, "C++ host behaviours")
        img = plugin.render_view(hnd, B.CloudSettings(global_scale=scale), B.headless_view(w, h), fmt="rgba8_srgb")
    finally:
        parts.destroy(); hnd.destroy()
    cpp = np.fromfile(raw_f, np.uint8).reshape(h, w, 4)
    assert np.array_equal(cpp, img)
    assert not np.array_equal(moved, cloud.position_visibility)
