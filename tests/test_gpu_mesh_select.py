"""bgs_cloud_select_in_mesh on the GPU: the inside mask bit for bit against the CPU oracle (select_oracle/) on every
mesh case and layout, the modes, both device copies of the lane, ordering against queued frames, and the errors."""
import ctypes as C

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import mesh_cases as MC
from bevy_gaussian_splatting_b200 import abi
from select_oracle import select_oracle as SO

pytestmark = pytest.mark.gpu

PIXEL_TOL = 1e-3
F = np.float32


@pytest.fixture(scope="module")
def plugin():
    p = B.GaussianSplattingPlugin(0)
    yield p
    p.destroy()


def cloud_at(pos_vis: np.ndarray, seed: int = 0) -> B.PlanarGaussian3d:
    c = B.random_gaussians_3d_seeded(len(pos_vis), seed)
    c.position_visibility[:] = pos_vis
    return c


def add(plugin, cloud, layout):
    return plugin.add_cloud(cloud, f16=layout == "f16", precompute_covariance=layout == "cov")


def transform() -> np.ndarray:
    M = np.eye(4)
    M[:3, :3] = MC.rotation(9) @ np.diag([1.3, 0.6, 1.7])
    M[:3, 3] = (0.2, -0.4, 0.1)
    return M.astype(F)


def oracle_mask(pos, mesh, M=None):
    m, s = SO.select_in_mesh(pos, *mesh, M, grid=True)
    if len(pos) * max(len(mesh[1]), 1) <= 2e8:                # (the CPU tests hold the grid to the brute force)
        mb, _ = SO.select_in_mesh(pos, *mesh, M)
        assert np.array_equal(m, mb)
    return m, s


def check(plugin, h, pos, mesh, M=None):
    """REPLACE: the lane equals the oracle's mask; the device's count equals the mask's."""
    want, n_want = oracle_mask(pos, mesh, M)
    got = plugin.select_in_mesh(h, *mesh, M)
    vis = plugin.visibility(h)
    assert np.array_equal(vis, want.astype(F)), f"mask differs at {np.flatnonzero(vis != want)[:8]}"
    assert got == n_want == int(want.sum())
    return want


@pytest.mark.parametrize("layout", ["f32", "f16", "cov"])
@pytest.mark.parametrize("n", [1, 31, 32, 1000, 200_000])
def test_mask_matches_oracle(plugin, layout, n):
    for name in sorted(MC.MESHES):
        mesh = MC.MESHES[name]()
        pos = MC.scatter(mesh, n, n % 7)
        if name == "box" and n >= 1000:
            pos[: len(MC.knife_points())] = MC.knife_points()
        h = add(plugin, cloud_at(pos), layout)
        try:
            for M in (None, transform()):
                check(plugin, h, pos, mesh, M)
        finally:
            h.destroy()


@pytest.mark.parametrize("offset", [0.0, 1e4])
def test_knife_points(plugin, offset):
    v, i = MC.box()
    v = (v + F(offset)).astype(F)
    pos = MC.knife_points(offset)
    h = plugin.add_cloud(cloud_at(pos))
    try:
        check(plugin, h, pos, (v, i))
    finally:
        h.destroy()


def test_six_million_against_the_box(plugin):
    cloud = B.random_gaussians_3d_seeded(6_000_000, 0)
    mesh = MC.box((-0.5, -0.7, -0.3), (0.6, 0.4, 0.8))
    h = plugin.add_cloud(cloud, f16=True)
    try:
        m = check(plugin, h, cloud.position_visibility, mesh)
        assert 0 < m.sum() < len(m)
    finally:
        h.destroy()


def test_a_million_against_a_sphere(plugin):
    cloud = B.random_gaussians_3d_seeded(1_000_000, 1)
    mesh = MC.icosphere(3, 0.8)                            # 1280 triangles
    h = plugin.add_cloud(cloud)
    try:
        m = check(plugin, h, cloud.position_visibility, mesh)
        assert 0 < m.sum() < len(m)
    finally:
        h.destroy()


def test_whole_cloud_in_one_cell(plugin):
    mesh = MC.big_and_small()
    pos = MC.pts(np.random.default_rng(2).uniform(-1e-4, 1e-4, (50_000, 3)) + (0.0, 0.31, 0.27))
    h = plugin.add_cloud(cloud_at(pos))
    try:
        check(plugin, h, pos, mesh)
    finally:
        h.destroy()


def test_empty_and_rejected_meshes(plugin):
    pos = MC.scatter(MC.box(), 5000, 3)
    h = plugin.add_cloud(cloud_at(pos))
    try:
        for mesh in (MC.all_rejected(), (np.zeros((0, 3), F), np.zeros((0, 3), np.uint32))):
            plugin.set_visibility(h, np.full(len(pos), 0.25, F))
            assert plugin.select_in_mesh(h, *mesh) == 0
            assert not plugin.visibility(h).any()
            plugin.set_visibility(h, np.full(len(pos), 0.25, F))
            assert plugin.select_in_mesh(h, *mesh, mode="add") == 0
            assert np.all(plugin.visibility(h) == F(0.25))
    finally:
        h.destroy()


def test_modes(plugin):
    pos = MC.scatter(MC.box(), 20_000, 4)
    a, b = MC.box((-1, -1, -1), (0.2, 0.3, 0.4)), MC.icosphere(2, 0.9)
    ma, _ = oracle_mask(pos, a)
    mb, _ = oracle_mask(pos, b)
    h = plugin.add_cloud(cloud_at(pos))
    try:
        labels = np.random.default_rng(5).choice(np.array([0.0, 0.25, 0.5, 2.0, 1.0], F), len(pos))
        plugin.set_visibility(h, labels)
        assert plugin.select_in_mesh(h, *a) == int(ma.sum())        # replace: 0 / 1 whatever was there
        assert np.array_equal(plugin.visibility(h), ma.astype(F))
        plugin.set_visibility(h, labels)
        plugin.select_in_mesh(h, *a, mode="add")                   # add: untouched outside, bit for bit
        v = plugin.visibility(h)
        assert np.all(v[ma] == 1.0) and np.array_equal(v[~ma].view(np.uint32), labels[~ma].view(np.uint32))
        plugin.select_in_mesh(h, *a)
        plugin.select_in_mesh(h, *b, mode="add")                   # two meshes: the oracle's OR
        assert np.array_equal(plugin.visibility(h), (ma | mb).astype(F))
        plugin.invert_selection(h)                                 # subtract b from (a | b): invert, add, invert
        plugin.select_in_mesh(h, *b, mode="add")
        plugin.invert_selection(h)
        assert np.array_equal(plugin.visibility(h), ((ma | mb) & ~mb).astype(F))
        with pytest.raises(ValueError):
            plugin.select_in_mesh(h, *a, mode="subtract")
    finally:
        h.destroy()


def oracle_frame(oracle, plugin, h, cloud, vis, settings, view, layout):
    oc = B.PlanarGaussian3d(cloud.position_visibility.copy(), cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity)
    oc.position_visibility[:, 3] = vis
    s_abi = settings.to_abi()
    if layout == "f16":
        oc = oc.rounded_to_f16()
    if layout == "cov":
        oc = oc.precomputed_covariance().rounded_to_f16()
        s_abi.reserved = 1
    return oracle.render_tiles(oc, view.to_abi(), plugin.cloud_uniform(settings, None, h.aabb), s_abi)


@pytest.mark.parametrize("layout", ["f32", "f16", "cov"])
def test_selection_updates_both_copies(plugin, oracle, layout):
    cloud = B.random_gaussians_3d_seeded(30000, 9)
    cloud.position_visibility[:, :3] *= np.float32(0.1)
    view = B.headless_view(320, 200)
    mesh = MC.icosphere(3, 1.2)
    h = add(plugin, cloud, layout)
    try:
        s_all = B.CloudSettings(global_scale=0.25, binning_rounds=False)
        plugin.render_view(h, s_all, view)
        before = plugin.render_view(h, s_all, view).copy()
        mask = check(plugin, h, cloud.position_visibility, mesh)
        assert 0.1 < mask.mean() < 0.9
        after = plugin.render_view(h, s_all, view)
        assert np.array_equal(after.view(np.uint32), before.view(np.uint32))
        for mode in (B.DrawMode.Selected, B.DrawMode.HighlightSelected):
            s = B.CloudSettings(global_scale=0.25, draw_mode=mode, binning_rounds=False)
            img = plugin.render_view(h, s, view)
            til = oracle_frame(oracle, plugin, h, cloud, mask.astype(F), s, view, layout)
            assert np.array_equal(plugin.tile_ranges(), til["tile_ranges"]), mode
            assert float(np.abs(img - til["image"]).max()) <= PIXEL_TOL
    finally:
        h.destroy()


def test_select_after_queued_frames(plugin, oracle):
    cloud = B.random_gaussians_3d_seeded(40000, 11)
    cloud.position_visibility[:, :3] *= np.float32(0.1)
    view = B.headless_view(320, 200)
    h = plugin.add_cloud(cloud)
    try:
        s = B.CloudSettings(global_scale=0.25, binning_rounds=False, draw_mode=B.DrawMode.Selected)
        for _ in range(4):
            plugin.render_view(h, s, view, asynchronous=True)
        mask = check(plugin, h, cloud.position_visibility, MC.box((-1, -1, -1), (0.5, 0.5, 0.5)))
        assert plugin.sync()
        img = plugin.render_view(h, s, view)
        til = oracle_frame(oracle, plugin, h, cloud, mask.astype(F), s, view, "f32")
        assert np.abs(img - til["image"]).max() <= PIXEL_TOL
    finally:
        h.destroy()


def test_select_on_a_cloud_another_context_has_queued(plugin, oracle):
    cloud = B.random_gaussians_3d_seeded(40000, 12)
    cloud.position_visibility[:, :3] *= np.float32(0.1)
    view = B.headless_view(320, 200)
    other = B.GaussianSplattingPlugin(0)
    h = plugin.add_cloud(cloud)
    try:
        s = B.CloudSettings(global_scale=0.25, binning_rounds=False, draw_mode=B.DrawMode.Selected)
        for _ in range(4):
            other.render_view(h, s, view, asynchronous=True)
        mask = check(plugin, h, cloud.position_visibility, MC.torus(32, 16))
        assert other.sync()
        img = other.render_view(h, s, view)
        til = oracle_frame(oracle, other, h, cloud, mask.astype(F), s, view, "f32")
        assert np.abs(img - til["image"]).max() <= PIXEL_TOL
    finally:
        h.destroy()
        other.destroy()


def test_debug_hooks_keep_the_last_frame(plugin):
    cloud = B.random_gaussians_3d_seeded(20000, 13)
    view = B.headless_view(320, 200)
    h = plugin.add_cloud(cloud)
    try:
        s = B.CloudSettings(global_scale=0.25, binning_rounds=False)
        plugin.render_view(h, s, view)
        stats0, se0, tr0 = plugin.frame_stats(), plugin.sorted_entries().copy(), plugin.tile_ranges().copy()
        plugin.select_in_mesh(h, *MC.icosphere(2, 1.5))
        stats1 = plugin.frame_stats()
        assert (stats1.n, stats1.n_visible, stats1.n_pairs) == (stats0.n, stats0.n_visible, stats0.n_pairs)
        assert np.array_equal(plugin.sorted_entries(), se0) and np.array_equal(plugin.tile_ranges(), tr0)
        plugin.stage_times_us()
    finally:
        h.destroy()


def test_errors(plugin):
    cloud = B.random_gaussians_3d_seeded(100, 0)
    h = plugin.add_cloud(cloud)
    lib, ctx = plugin._lib, plugin._ctx
    v, i = MC.box()
    vp, ip = v.ctypes.data_as(C.c_void_p), i.ctypes.data_as(C.c_void_p)
    n_in = C.c_uint32()
    try:
        plugin.set_visibility(h, np.full(100, 0.5, F))
        calls = [
            lambda: lib.bgs_cloud_select_in_mesh(None, h._h, vp, 8, ip, 12, None, 0, C.byref(n_in)),
            lambda: lib.bgs_cloud_select_in_mesh(ctx, None, vp, 8, ip, 12, None, 0, C.byref(n_in)),
            lambda: lib.bgs_cloud_select_in_mesh(ctx, h._h, None, 8, ip, 12, None, 0, C.byref(n_in)),
            lambda: lib.bgs_cloud_select_in_mesh(ctx, h._h, vp, 8, None, 12, None, 0, C.byref(n_in)),
            lambda: lib.bgs_cloud_select_in_mesh(ctx, h._h, vp, 7, ip, 12, None, 0, C.byref(n_in)),   # index 7 >= 7
            lambda: lib.bgs_cloud_select_in_mesh(ctx, h._h, vp, 8, ip, 12, None, 2, C.byref(n_in)),   # unknown mode
        ]
        for call in calls:
            assert call() == abi.BGS_EINVAL
        assert np.all(plugin.visibility(h) == F(0.5))                # a refused call changed nothing
        assert lib.bgs_cloud_select_in_mesh(ctx, h._h, None, 0, None, 0, None, 0, None) == abi.BGS_OK   # nt == 0, NULL out
        assert not plugin.visibility(h).any()
        assert lib.bgs_cloud_select_in_mesh(ctx, h._h, vp, 8, ip, 12, None, 0, None) == abi.BGS_OK
        with pytest.raises(ValueError):
            plugin.select_in_mesh(h, v[:, :2], i)
        with pytest.raises(ValueError):
            plugin.select_in_mesh(h, v, i.reshape(-1))
    finally:
        h.destroy()


def test_cloud_on_another_device_is_refused():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    p0, p1 = B.GaussianSplattingPlugin(0), B.GaussianSplattingPlugin(1)
    h = p1.add_cloud(B.random_gaussians_3d_seeded(100, 0))
    try:
        with pytest.raises(abi.BgsError) as e:
            p0.select_in_mesh(h, *MC.box())
        assert e.value.status == abi.BGS_EINVAL
    finally:
        h.destroy()
        p0.destroy()
        p1.destroy()
