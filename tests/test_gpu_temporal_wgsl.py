"""Gaussian4d records on the H100 held to the INDEPENDENT float64 restatement of the reference (tests/wgsl_emu_4d.py)
directly, not only through temporal_oracle/.

* project_4d_kernel (bgs_render_4d), project_4d_scene_kernel (bgs_render_scene_4d) and project_4d_many_kernel
  (bgs_render_entities_many); the scene paths list one 4D cloud twice, at different times and windows.
* Decisions and geometry as in tests/test_wgsl_restatement_4d.py: equal unless the float64 margin lies inside the f32
  error bound; values within the running error bounds of temporal_wgsl_cases.
* SH-based colours within the bound with gpu=True, which names each source of error: rsqrt.approx (2 ulp) in every
  normalisation, the FMA sums (covered by the unfused bound) and __powf's lg2 / ex2 approximations in the sRGB decode.
* Large theta: the time terms follow det_cos's documented bound of the true cosine up to |4 pi theta| ~ 1.3e10.
* Small whole frames (Color and Velocity, OBB and AABB) against the emulator's quad walk, every pixel within the bound
  temporal_wgsl_cases.check_frame derives from the record bounds, with the blend's ex2.approx added.
Velocity is 0 for every input here (transpose(M) * M is diagonal, so delta_mean is 0; see temporal_wgsl_cases.edge_cloud):
the Velocity cases check the time mask, both frustum tests, the geometry and the zero colour and opacity, not a
non-zero velocity (tests/test_gpu_temporal.py holds those to the oracle bit for bit).
"""
import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import temporal_wgsl_cases as TW
from bevy_gaussian_splatting_b200.plugin import CloudTransform
from oracle import oracle as O

pytestmark = pytest.mark.gpu

f32 = np.float32
RM = B.RasterizeMode
W, H = 160, 112
PREV_EYE = (2.3, 1.7, 4.6)


@pytest.fixture(scope="module")
def plugin():
    p = B.GaussianSplattingPlugin(0)
    yield p
    p.destroy()


def settings(mode, t=0.5, window=(0.0, 1.0), **kw):
    return B.CloudSettings(gaussian_mode=B.GaussianMode.Gaussian4d, rasterize_mode=mode, time=t, num_classes=3,
                           global_scale=1.3, global_opacity=0.9, time_start=window[0], time_stop=window[1], **kw)


def prev_view(view):
    return B.perspective_view(PREV_EYE, (0.1, 0.0, -0.2), view.width, view.height, up=(0.15, 1.0, -0.05))


def render4(plugin, h, s, view, tr):
    flow = s.rasterize_mode == RM.OpticalFlow
    pv, dt = (prev_view(view), 1 / 30) if flow else (None, None)
    img = plugin.render_view(h, s, view, transform=tr, previous_view=pv, delta_time=dt)
    u, _, ex = plugin._call_args(h, s, tr, previous_view=pv, delta_time=dt)
    return img, u, ex


def sorted_ids(cloud, view, u):
    return O.radix_sort(O.keygen(cloud.position_visibility, view.to_abi(), u, 32), 32)[1]


CASES = [(m, aabb, cs) for m in [RM.Color, RM.Classification, RM.Depth, RM.Position, RM.OpticalFlow, RM.Velocity]
         for aabb, cs in ((False, 0), (True, 1))]


@pytest.mark.parametrize("mode,aabb,cs", CASES, ids=[f"{m.name}-{'aabb' if a else 'obb'}-cs{c}" for m, a, c in CASES])
def test_project_4d_kernel_against_wgsl(plugin, mode, aabb, cs):
    cloud = TW.edge_cloud(512, 21)
    view = TW.off_axis_view(W, H)
    tr = CloudTransform(TW.model_matrix())
    h = plugin.add_cloud(cloud)
    try:
        s = settings(mode, aabb=aabb, color_space=B.GaussianColorSpace(cs))
        _, u, ex = render4(plugin, h, s, view, tr)
        rec, ids = plugin.projected()
        compared, undecided, expected = TW.check_records(rec, ids, cloud, view, u, s, (0.0, 1.0), sorted_ids(cloud, view, u),
                                                         ex, gpu=True)
        assert compared >= 100 and undecided <= 2 * expected + 4, (compared, undecided, expected)
    finally:
        h.destroy()


def _scene_check(plugin, render, mode):
    """One 4D cloud listed twice at different times and windows: each entity's slice of the records against the
    emulator with that entity's uniform and window."""
    cloud = TW.edge_cloud(256, 23)
    view = TW.off_axis_view(W, H)
    tr = CloudTransform(TW.model_matrix())
    h = plugin.add_cloud(cloud)
    try:
        sts = [settings(mode, 0.5, (0.0, 1.0)), settings(mode, 0.42, (-0.5, 2.0))]
        ents = [(h, st, tr) for st in sts]
        render(ents, view)
        rec, ids = plugin.projected()
        n = len(cloud)
        total = 0
        for j, st in enumerate(sts):
            u = plugin.cloud_uniform(st, tr, h.aabb)
            sel = (ids // n) == j
            compared, undecided, expected = TW.check_records(rec[sel], ids[sel] - j * n, cloud, view, u, st,
                                                             (st.time_start, st.time_stop), None, None, gpu=True)
            assert undecided <= 2 * expected + 4, (j, undecided, expected)
            total += compared
        assert total >= 200
    finally:
        h.destroy()


@pytest.mark.parametrize("mode", [RM.Color, RM.Position, RM.Velocity])
def test_project_4d_scene_kernel_against_wgsl(plugin, mode):
    _scene_check(plugin, plugin.render_scene, mode)


@pytest.mark.parametrize("mode", [RM.Color, RM.Velocity])
def test_project_4d_many_kernel_against_wgsl(plugin, mode):
    _scene_check(plugin, plugin.render_entities_many, mode)


def test_large_theta_time_terms(plugin):
    """theta from 1 to 1e9 by half decades, both signs (|2 pi theta| up to 6.3e9, |4 pi theta| up to 1.3e10): the
    kernel's colour within the gpu bound, whose time terms carry det_cos_bound(arg) around math.cos of WGSL's f32
    argument."""
    thetas = [s * 10.0 ** e for e in np.arange(0.0, 9.25, 0.5) for s in (1.0, -1.0)]
    cloud = TW.theta_cloud(thetas, seed=9)
    view = TW.off_axis_view(W, H)
    tr = CloudTransform(TW.model_matrix())
    h = plugin.add_cloud(cloud)
    try:
        s = settings(RM.Color, color_space=B.GaussianColorSpace.LinRec709Display)
        _, u, _ = render4(plugin, h, s, view, tr)
        rec, ids = plugin.projected()
        compared, undecided, expected = TW.check_records(rec, ids, cloud, view, u, s, (0.0, 1.0), None, None, gpu=True)
        assert compared >= len(thetas) - 4 and undecided <= 2 * expected + 2
        assert np.abs(cloud.timestamp_timescale[ids, 0] - 0.5).max() >= 0.99e9
    finally:
        h.destroy()


@pytest.mark.parametrize("mode,aabb", [(RM.Color, False), (RM.Color, True), (RM.Velocity, False), (RM.Velocity, True)])
def test_small_frames_against_wgsl_walk(plugin, mode, aabb):
    """63 splats: the kernel's frame against the emulator's quad walk within check_frame's derived per-pixel bound;
    the undecided decisions within twice the predicted count plus four (as in test_wgsl_restatement_4d)."""
    cloud = TW.edge_cloud(72, 7)
    cloud = cloud.subset(np.flatnonzero(np.arange(72) % 8 != 2))     # not the rows built on the time threshold
    view = TW.off_axis_view(96, 64)
    tr = CloudTransform(TW.model_matrix())
    h = plugin.add_cloud(cloud)
    try:
        s = settings(mode, aabb=aabb, color_space=B.GaussianColorSpace.LinRec709Display, binning_rounds=False)
        img, u, _ = render4(plugin, h, s, view, tr)
        rec, ids = plugin.projected()
        order = TW.frame_order(cloud, view, u)
        bounds = {}
        _, rec_undecided, rec_expected = TW.check_records(rec, ids, cloud, view, u, s, (0.0, 1.0), None, None, gpu=True,
                                                          bounds=bounds)
        assert rec_undecided <= 2 * rec_expected + 4
        sh4 = TW.shader_for(view, u, s, (0.0, 1.0))
        compared, undecided, expected, want = TW.check_frame(img, cloud, sh4, order, rec, ids, bounds, gpu=True)
        if mode == RM.Color:
            assert (np.nan_to_num(want).max(axis=2) > 0.02).sum() >= 100
        assert undecided <= 2 * expected + 4, (undecided, expected)
        assert compared >= 0.9 * view.width * view.height
    finally:
        h.destroy()
