"""Gaussian4d clouds on the GPU (bgs_cloud_upload_4d, bgs_render_4d, project_4d_kernel) against temporal_oracle/.

* Records (bgs_debug_projected) by front-to-back rank, OBB and AABB, every accepted RasterizeMode, every draw mode,
  several times: rank -> index, centre, uv rows, bbox, opacity (so the time mask and the moved frustum test) bit for
  bit; Velocity, OpticalFlow, Depth and Position colours bit for bit; Color and Classification colours within a bound
  of the SH sums' magnitude (the kernel fuses them and uses rsqrt.approx and an approximate pow).
* Sorted entries equal those of a 3D cloud of the same positions (key-gen does not depend on time).
* Whole frames within 1e-3 of the oracle's tile walk; queued, sort-all and chunked frames equal the synchronous one
  byte for byte; a depth-tested frame's splat depths (from the moved positions) equal the oracle's bit for bit.
* Upload -> download bit for bit; subsets in both modes; selection and particle steps on a 4D cloud equal those on the
  3D cloud of the same positions.
* Refusals return BGS_EINVAL and change nothing: launch count and target bytes.
"""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import project_cases as PC
import temporal_cases as TC
from bevy_gaussian_splatting_b200 import abi
from temporal_oracle import temporal_oracle as T

pytestmark = pytest.mark.gpu

f32 = np.float32
RM = B.RasterizeMode
MODES = [RM.Color, RM.Depth, RM.Position, RM.Classification, RM.OpticalFlow, RM.Velocity]
EXACT = {RM.Depth, RM.Position, RM.OpticalFlow, RM.Velocity}


@pytest.fixture(scope="module")
def plugin():
    p = B.GaussianSplattingPlugin(0)
    yield p
    p.destroy()


@pytest.fixture(scope="module")
def scene():
    return TC.scene_4d(3000, 5, selected=True)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same(got, want):
    """Bit for bit, a NaN's payload aside (project_cases.bits_agree: x86 and CUDA make different NaNs)."""
    return bool(PC.bits_agree(got, want).all())


def moved_view(view, d=(0.03, -0.02, 0.05)):
    eye = np.asarray(view.world_position, np.float64) + d
    return B.perspective_view(tuple(eye), tuple(eye + (0.0, -0.3, -1.0)), view.width, view.height)


def settings(mode, t, **kw):
    return B.CloudSettings(gaussian_mode=B.GaussianMode.Gaussian4d, rasterize_mode=mode, time=t, num_classes=3, **kw)


def render(plugin, h, s, view, **kw):
    prev = moved_view(view) if s.rasterize_mode == RM.OpticalFlow else None
    return plugin.render_view(h, s, view, previous_view=prev, delta_time=1 / 30 if prev else None, **kw)


def oracle_frame(cloud, s, view, plugin, h, **kw):
    u, st, ex = plugin._call_args(h, s, None, previous_view=moved_view(view) if s.rasterize_mode == RM.OpticalFlow else None,
                                  delta_time=1 / 30 if s.rasterize_mode == RM.OpticalFlow else None)
    if ex is None:
        ex = abi.bgs_render_extras(num_classes=int(s.num_classes))
    return T.frame(cloud, view.to_abi(), u, st, s.time_start, s.time_stop, extras=ex, **kw)


def sh_bound(cloud, ids):
    """|colour - oracle colour| bound: 2e-5 of the SH sums' magnitude (basis terms <= 3 each), x 2.4 for the decode."""
    mag = f32(0.5) + 3.0 * np.abs(cloud.spherindrical_harmonic[ids]).reshape(-1, 48, 3).sum(1)
    return 2.4 * 2e-5 * mag + 1e-6


@pytest.mark.parametrize("aabb", [False, True])
@pytest.mark.parametrize("mode", MODES)
def test_records_against_oracle(plugin, scene, mode, aabb):
    view = B.headless_view(160, 112)
    h = plugin.add_cloud(scene)
    try:
        for t, draw, cs in ((0.15, B.DrawMode.All, 0), (0.5, B.DrawMode.Selected, 1), (0.85, B.DrawMode.HighlightSelected, 0)):
            s = settings(mode, t, aabb=aabb, draw_mode=draw, color_space=B.GaussianColorSpace(cs))
            render(plugin, h, s, view)
            rec, ids = plugin.projected()
            o = oracle_frame(scene, s, view, plugin, h, want_image=False)
            assert np.array_equal(ids, o["rank_to_id"])
            geo = [0, 1, 2, 3, 4, 5, 6, 7, 11]
            assert same(rec[:, geo], o["records"][:, geo]), (mode, aabb, t)
            bb = rec[:, 6:8].view(np.uint32)
            drawn = ((bb[:, 0] & 0xFFFF) <= (bb[:, 0] >> 16)) & ((bb[:, 1] & 0xFFFF) <= (bb[:, 1] >> 16))
            assert 0 < drawn.sum() < len(rec)   # some splats are masked by time at every t
            if mode in EXACT:
                assert same(rec[:, 8:11], o["records"][:, 8:11])
            else:
                err = np.abs(rec[drawn, 8:11].astype(np.float64) - o["records"][drawn, 8:11])
                assert (err <= sh_bound(scene, ids[drawn])).all(), err.max()
    finally:
        h.destroy()


def test_velocity_records_of_moving_splats(plugin):
    """Splats whose Velocity is not 0 (temporal_cases.fast_arrays): colours and zero opacities bit for bit."""
    rot8, so, tt, t = TC.fast_arrays(4000, 7)
    rng = np.random.default_rng(7)
    pos = (rng.random((4000, 3), np.float32) - 0.5) * f32(3.0)
    c = TC.cloud_4d(pos, rot8=rot8, so=so, tt=tt, seed=7)
    view = B.headless_view(128, 96)
    h = plugin.add_cloud(c)
    try:
        s = settings(RM.Velocity, float(t))
        render(plugin, h, s, view)
        rec, ids = plugin.projected()
        o = oracle_frame(c, s, view, plugin, h, want_image=False)
        assert np.array_equal(ids, o["rank_to_id"]) and same(rec, o["records"])
        bb = rec[:, 6:8].view(np.uint32)
        drawn = (bb[:, 0] & 0xFFFF) <= (bb[:, 0] >> 16)
        assert (drawn & (rec[:, 11] > 0)).any() and (drawn & (rec[:, 11] == 0)).any()
    finally:
        h.destroy()


def test_sorted_entries_are_the_3d_ones(plugin, scene):
    view = B.headless_view(128, 96)
    h4 = plugin.add_cloud(scene)
    c3 = B.random_gaussians_3d_seeded(len(scene), 1)
    c3 = B.PlanarGaussian3d(scene.position_visibility, c3.spherical_harmonic, c3.rotation, c3.scale_opacity)
    h3 = plugin.add_cloud(c3)
    try:
        for bits_ in (B.RadixSortDepthBits.Bits16, B.RadixSortDepthBits.Bits32):
            for sort_all in (False, True):
                render(plugin, h4, settings(RM.Color, 0.4, radix_sort_depth_bits=bits_, sort_all=sort_all), view)
                e4 = plugin.sorted_entries()
                plugin.render_view(h3, B.CloudSettings(radix_sort_depth_bits=bits_, sort_all=sort_all), view)
                assert np.array_equal(e4, plugin.sorted_entries())
    finally:
        h4.destroy(); h3.destroy()


@pytest.mark.parametrize("mode", [RM.Color, RM.Velocity, RM.Position])
def test_frames_against_oracle_walk(plugin, scene, mode):
    view = B.headless_view(160, 112)
    h = plugin.add_cloud(scene)
    try:
        for aabb in (False, True):
            s = settings(mode, 0.45, aabb=aabb, color_space=B.GaussianColorSpace.LinRec709Display, binning_rounds=False)
            img = render(plugin, h, s, view)
            o = oracle_frame(scene, s, view, plugin, h)
            assert np.abs(img - o["image"]).max() <= 1e-3
            # queued, sort-all and chunked frames: byte for byte the synchronous one
            for kw, s2 in ((dict(asynchronous=True), s), ({}, dataclasses.replace(s, sort_all=True)),
                           ({}, dataclasses.replace(s, binning_rounds=True))):
                out = render(plugin, h, s2, view, **kw)
                if kw:
                    assert plugin.sync()
                assert out.tobytes() == img.tobytes(), kw
    finally:
        h.destroy()


def test_depth_tested_frame(plugin, scene):
    torch = pytest.importorskip("torch")
    view = B.headless_view(128, 96)
    h = plugin.add_cloud(scene)
    try:
        s = settings(RM.Color, 0.6, color_space=B.GaussianColorSpace.LinRec709Display, binning_rounds=False)
        rng = np.random.default_rng(3)
        zs = rng.uniform(0.0, 0.02, (96, 128)).astype(np.float32)
        zd = torch.from_numpy(zs).cuda()
        torch.cuda.synchronize()
        img = render(plugin, h, s, view, scene_depth=zd)
        o = oracle_frame(scene, s, view, plugin, h, scene=zs)
        d = plugin.splat_depths()
        assert same(d, o["depths"])
        assert np.abs(img - o["image"]).max() <= 1e-3
        plain = render(plugin, h, s, view)
        assert plain.tobytes() != img.tobytes()   # the test hides something
    finally:
        h.destroy()


def test_upload_download_subset(plugin, scene):
    h = plugin.add_cloud(scene)
    try:
        planes = plugin.download_planes(h)
        for a, b in zip(planes, scene.planes()):
            assert a.tobytes() == b.tobytes()
        idx = np.array([5, 0, 17, 17, 2999], np.uint32)
        sub = plugin.subset(h, idx)
        for a, b in zip(plugin.download_planes(sub), scene.subset(idx).planes()):
            assert a.tobytes() == b.tobytes()
        sub.destroy()
        sel = plugin.subset(h)   # selection mode: visibility >= 0.5
        keep = np.flatnonzero(~(scene.position_visibility[:, 3] < 0.5))
        for a, b in zip(plugin.download_planes(sel), scene.subset(keep).planes()):
            assert a.tobytes() == b.tobytes()
        # a subset renders like a fresh upload of the same gaussians
        view = B.headless_view(96, 64)
        fresh = plugin.add_cloud(scene.subset(keep))
        s = settings(RM.Color, 0.3)
        a = render(plugin, sel, s, view)
        assert a.tobytes() == render(plugin, fresh, s, view).tobytes()
        sel.destroy(); fresh.destroy()
    finally:
        h.destroy()


def test_selection_and_particles_as_3d(plugin, scene):
    c3 = B.PlanarGaussian3d(scene.position_visibility, np.zeros((len(scene), 48), np.float32),
                            scene.isotropic_rotations[:, :4], scene.scale_opacity)
    h4, h3 = plugin.add_cloud(scene), plugin.add_cloud(c3)
    try:
        q = B.SparseSelect(0.05, 3)
        assert plugin.select_sparse(h4, q) == plugin.select_sparse(h3, q)
        assert plugin.visibility(h4).tobytes() == plugin.visibility(h3).tobytes()
        beh = B.random_particle_behaviors(len(scene), 1)
        for h in (h4, h3):
            p = plugin.add_particles(beh)
            plugin.step_particles(h, p, 1 / 60)
            plugin.sync()
            p.destroy()
        assert plugin.positions(h4).tobytes() == plugin.positions(h3).tobytes()
        # a stepped 4D cloud renders from its moved base positions
        render(plugin, h4, settings(RM.Color, 0.5), B.headless_view(64, 48))
    finally:
        h4.destroy(); h3.destroy()


def _call4(plugin, h, st, view, u=None, ts=0.0, te=1.0, ex=None, out=None):
    v = view.to_abi()
    u = u if u is not None else plugin.cloud_uniform(B.CloudSettings())
    return plugin._lib.bgs_render_4d(plugin._ctx, h._h, C.byref(v), C.byref(u), C.byref(st),
                                     None if ex is None else C.byref(ex), None, out.ctypes.data_as(C.c_void_p), 2, 0,
                                     C.c_float(ts), C.c_float(te))


def test_refusals_change_nothing(plugin, scene):
    view = B.headless_view(96, 64)
    h4 = plugin.add_cloud(scene)
    h3 = plugin.add_cloud(B.random_gaussians_3d_seeded(2000, 1))
    try:
        s = settings(RM.Color, 0.5)
        out = render(plugin, h4, s, view)
        launches, before = plugin.last_launch_count, out.copy()
        good = s.to_abi()
        bad = []
        for ts, te in ((0.5, 0.5), (0.0, float("inf")), (float("nan"), 1.0), (-3e38, 3e38)):
            bad.append((h4, good, None, ts, te))
        for t in (float("nan"), float("inf")):
            u = plugin.cloud_uniform(dataclasses.replace(s, time=t))
            bad.append((h4, good, u, 0.0, 1.0))
        normal = s.to_abi(); normal.rasterize_mode = int(RM.Normal)
        mode7 = s.to_abi(); mode7.rasterize_mode = 7
        g3 = s.to_abi(); g3.gaussian_mode = 1
        bad += [(h4, normal, None, 0.0, 1.0), (h4, mode7, None, 0.0, 1.0), (h4, g3, None, 0.0, 1.0), (h3, good, None, 0.0, 1.0)]
        for h, st, u, ts, te in bad:
            assert _call4(plugin, h, st, view, u, ts, te, out=out) == abi.BGS_EINVAL
            assert plugin.last_launch_count == launches and out.tobytes() == before.tobytes()
        # the 3D calls refuse a 4D cloud; bgs_render_aux too; interpolation of 4D clouds
        v, u3 = view.to_abi(), plugin.cloud_uniform(B.CloudSettings())
        s3 = B.CloudSettings().to_abi()
        assert plugin._lib.bgs_render(plugin._ctx, h4._h, C.byref(v), C.byref(u3), C.byref(s3), out.ctypes.data_as(C.c_void_p), 2, 0) == abi.BGS_EINVAL
        with pytest.raises(abi.BgsError):
            plugin.render_view_aux(h4, B.CloudSettings(), view)
        other = plugin.add_cloud(scene)
        dst = plugin.add_cloud(scene)
        with pytest.raises(abi.BgsError):
            plugin.interpolate(dst, h4, other, B.CloudSettings(time=0.5))
        other.destroy(); dst.destroy()
        with pytest.raises(abi.BgsError):   # the download call of another layout
            pos = np.empty((len(scene), 4), np.float32)
            sh, rot, so = np.empty((len(scene), 48), np.float32), np.empty((len(scene), 4), np.float32), np.empty((len(scene), 4), np.float32)
            plugin._check(plugin._lib.bgs_cloud_download_f32(plugin._ctx, h4._h, *(a.ctypes.data_as(C.c_void_p) for a in (pos, sh, rot, so))))
        assert plugin.last_launch_count == launches and out.tobytes() == before.tobytes()
    finally:
        h4.destroy(); h3.destroy()


def test_mask_threshold_records(plugin):
    """Timescales walked ulp by ulp across marginal_t = 0.05: the draw decision and every record bit for bit.  (No f32
    input of det_exp gives 0.05f itself: near ln 0.05 its outputs step by about 3 ulps and skip it.)"""
    n = 257
    dt = f32(0.5)
    st0 = f32(float(dt) / np.sqrt(2 * np.log(20.0)))
    st = (np.array([st0], np.float32).view(np.int32).astype(np.int64) + np.arange(-128, 129)).astype(np.int32).view(np.float32)
    rot8 = np.tile(np.array([1, 0, 0, 0, 1, 0, 0, 0], np.float32), (n, 1))
    so = np.tile(np.array([0.05, 0.04, 0.03, 0.6], np.float32), (n, 1))
    tt = np.stack([np.zeros(n, np.float32), st, np.zeros(n, np.float32), np.zeros(n, np.float32)], 1)
    _, _, marg, mask = TC.condition(rot8, so, tt, 1.0, dt)
    assert mask.any() and (~mask).any()
    xs = np.linspace(-1.5, 1.5, n, dtype=np.float32)
    c = TC.cloud_4d(np.stack([xs, np.zeros(n, np.float32), np.zeros(n, np.float32)], 1), rot8=rot8, so=so, tt=tt)
    view = B.headless_view(256, 64)
    h = plugin.add_cloud(c)
    try:
        s = settings(RM.Color, float(dt))
        render(plugin, h, s, view)
        rec, ids = plugin.projected()
        o = oracle_frame(c, s, view, plugin, h, want_image=False)
        geo = [0, 1, 2, 3, 4, 5, 6, 7, 11]
        assert np.array_equal(ids, o["rank_to_id"]) and same(rec[:, geo], o["records"][:, geo])
        bb = rec[:, 6:8].view(np.uint32)
        drawn = (bb[:, 0] & 0xFFFF) <= (bb[:, 0] >> 16)
        assert np.array_equal(drawn, mask[ids])
    finally:
        h.destroy()
