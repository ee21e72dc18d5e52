"""bgs_cloud_select_sparse / bgs_cloud_visibility_get / _set on the GPU: SparseSelect's mask bit for bit against the
CPU oracle (select_oracle/), both device copies of the visibility lane updated (frames rendered after an edit match
the oracle's render of the host cloud with that visibility), and the ordering against queued frames."""
import ctypes as C

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import select_cases as SC
from bevy_gaussian_splatting_b200 import abi
from select_oracle import select_oracle as SO

pytestmark = pytest.mark.gpu

PIXEL_TOL = 1e-3


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


def oracle_mask(pos, radius, thr):
    m, s = SO.select_sparse(pos, radius, thr, grid=True)
    if len(pos) <= 20000:
        mb, _ = SO.select_sparse(pos, radius, thr)
        assert np.array_equal(m, mb)
    return m, s


def check_select(plugin, h, pos, radius, thr):
    want, n_want = oracle_mask(pos, radius, thr)
    got = plugin.select_sparse(h, B.SparseSelect(radius, thr))
    vis = plugin.visibility(h)
    assert np.array_equal(vis, want.astype(np.float32)), \
        f"mask differs at {np.flatnonzero(vis != want)[:8]} (n {len(pos)}, radius {radius}, threshold {thr})"
    assert got == n_want == int(want.sum())
    return want


def radii_for(n: int):
    """Uniform cloud in a 40^3 box: radii giving ~0.001, ~1 and ~30 expected neighbours."""
    rho = n / 40.0 ** 3
    return [float((k / rho / (4.0 / 3.0 * np.pi)) ** (1.0 / 3.0)) for k in (0.001, 1.0, 30.0)]


@pytest.mark.parametrize("layout", ["f32", "f16", "cov"])
@pytest.mark.parametrize("n", [1, 31, 32, 1000, 200_000])
def test_mask_matches_oracle(plugin, layout, n):
    cloud = B.random_gaussians_3d_seeded(n, n % 5)
    h = add(plugin, cloud, layout)
    try:
        for radius in radii_for(n):
            for thr in (1, 3, 32):
                check_select(plugin, h, cloud.position_visibility, radius, thr)
    finally:
        h.destroy()


@pytest.mark.parametrize("n,kind,layout", [(1_000_000, "uniform", "f16"), (1_000_000, "uniform", "f32"),
                                           (2_000_000, "clustered", "f16")])
def test_mask_matches_oracle_large(plugin, n, kind, layout):
    cloud = B.random_gaussians_3d_seeded(n, 7)
    if kind == "clustered":
        cloud.position_visibility[:] = SC.clustered(n, 7, clusters=4096, sigma=0.1)
    h = add(plugin, cloud, layout)
    try:
        radii = radii_for(n) if kind == "uniform" else [0.01, 0.05, 0.2]
        for radius in radii:
            for thr in (3, 32):
                check_select(plugin, h, cloud.position_visibility, radius, thr)
    finally:
        h.destroy()


@pytest.mark.parametrize("name", ["duplicates", "non_finite", "large_coordinates", "ply_padding", "knife_edge"])
def test_mask_matches_oracle_special_inputs(plugin, name, tmp_path):
    radii = (0.0, 0.05, 0.3, 1.0)
    if name == "duplicates":
        pos = SC.with_duplicates(3000, 12)
    elif name == "non_finite":
        pos = SC.non_finite(3000, 13)
    elif name == "large_coordinates":
        pos, radii = SC.large_coordinates(4000, 14), (1e-3, 0.05, 1e-12)
    elif name == "ply_padding":
        c = B.random_gaussians_3d_seeded(1000, 4)
        c.position_visibility[:, :3] *= np.float32(0.05)
        B.io.write_ply_3d(str(tmp_path / "c.ply"), c)
        pos = B.parse_ply_3d(str(tmp_path / "c.ply")).position_visibility
    else:
        pos, where, r = SC.knife_edge_cloud(0.1768)
        assert len(where) == 9
        radii = (r,)
    h = plugin.add_cloud(cloud_at(pos))
    try:
        for radius in radii:
            for thr in (0, 1, 2, 3, 64):
                m = check_select(plugin, h, pos, radius, thr)
                if name == "knife_edge" and thr == 2:
                    for (geo, kind), (i, j) in where.items():
                        assert m[i] == m[j] == (kind != "below"), (geo, kind)
    finally:
        h.destroy()


def test_repeated_buckets_are_scanned_once(plugin):
    """The 27-cell scan meets one bucket twice (asserted with the restated hash): the GPU must count it once.
    (A kernel without the bucket dedupe fails here.)"""
    pos, case = SC.repeated_bucket_cloud()
    assert SC.num_buckets(len(pos)) == 1024
    c_self = SC.cell_of(pos[case["self"]], 1.0)
    nbk = SC.neighbour_buckets(c_self, 1024)
    assert nbk.count(nbk[13]) > 1
    i, j = case["pair"]
    nbk = SC.neighbour_buckets(SC.cell_of(pos[i], 1.0), 1024)
    assert nbk.count(SC.bucket_of(SC.cell_of(pos[j], 1.0), 1024)) > 1
    h = plugin.add_cloud(cloud_at(pos))
    try:
        m2 = check_select(plugin, h, pos, 1.0, 2)
        assert m2[case["self"]] and not m2[i]
        m3 = check_select(plugin, h, pos, 1.0, 3)
        assert m3[i] and m3[j]
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


def check_frames(plugin, oracle, h, cloud, vis, view, layout):
    for mode in (B.DrawMode.Selected, B.DrawMode.HighlightSelected):
        s = B.CloudSettings(global_scale=0.25, draw_mode=mode, binning_rounds=False)
        img = plugin.render_view(h, s, view)
        til = oracle_frame(oracle, plugin, h, cloud, vis, s, view, layout)
        assert np.array_equal(plugin.tile_ranges(), til["tile_ranges"]), mode
        err = float(np.abs(img - til["image"]).max())
        assert err <= PIXEL_TOL, (mode, err)


@pytest.mark.parametrize("layout", ["f32", "f16", "cov"])
def test_selection_updates_both_copies(plugin, oracle, layout):
    cloud = B.random_gaussians_3d_seeded(30000, 9)
    cloud.position_visibility[:, :3] *= np.float32(0.1)       # +-2: a few neighbours each within 0.1
    view = B.headless_view(320, 200)
    h = add(plugin, cloud, layout)
    try:
        s_all = B.CloudSettings(global_scale=0.25, binning_rounds=False)
        plugin.render_view(h, s_all, view)
        before = plugin.render_view(h, s_all, view).copy()
        mask = check_select(plugin, h, cloud.position_visibility, 0.1, 3)
        assert 0.2 < mask.mean() < 0.8
        # DrawMode::All ignores the lane: bit-identical, and the hints the frame plans from survived the selection
        after = plugin.render_view(h, s_all, view)
        assert np.array_equal(after.view(np.uint32), before.view(np.uint32))
        # the lane the projection reads (block copy) holds the selection
        check_frames(plugin, oracle, h, cloud, mask.astype(np.float32), view, layout)
    finally:
        h.destroy()


def test_visibility_set_apply_invert_roundtrip(plugin, oracle):
    cloud = B.random_gaussians_3d_seeded(20000, 10)
    view = B.headless_view(256, 160)
    h = plugin.add_cloud(cloud, f16=True)
    try:
        rng = np.random.default_rng(0)
        idx = np.sort(rng.choice(len(cloud), 7000, replace=False)).astype(np.uint32)
        plugin.apply_selection(h, idx)
        assert np.array_equal(plugin.selection(h), idx)
        want = np.zeros(len(cloud), np.float32)
        want[idx] = 1.0
        assert np.array_equal(plugin.visibility(h), want)
        check_frames(plugin, oracle, h, cloud, want, view, "f16")
        plugin.invert_selection(h)
        assert np.array_equal(plugin.visibility(h), 1.0 - want)
        check_frames(plugin, oracle, h, cloud, 1.0 - want, view, "f16")
        labels = rng.choice(np.array([0.0, 0.25, 0.5, 0.75, 1.0, 2.0], np.float32), len(cloud))
        plugin.set_visibility(h, labels)
        assert np.array_equal(plugin.visibility(h), labels)
        check_frames(plugin, oracle, h, cloud, labels, view, "f16")
        assert np.array_equal(plugin.selection(h), np.flatnonzero(labels >= 0.5))
        plugin.invert_selection(h)                              # == 0 -> 1, everything else -> 0
        assert np.array_equal(plugin.visibility(h), (labels == 0).astype(np.float32))
        with pytest.raises(IndexError):
            plugin.apply_selection(h, [len(cloud)])
        # a selected subset of the host cloud (save_selection's cloud.subset(indices))
        sub = cloud.subset(idx)
        assert len(sub) == len(idx) and np.array_equal(sub.position_visibility, cloud.position_visibility[idx])
        assert len(cloud.subset(5)) == 5
    finally:
        h.destroy()


def test_visibility_lane_at_two_million(plugin):
    cloud = B.random_gaussians_3d_seeded(2_000_000, 3)
    h = plugin.add_cloud(cloud)
    try:
        v = (np.arange(len(cloud)) % 3 == 0).astype(np.float32)
        plugin.set_visibility(h, v)
        assert np.array_equal(plugin.visibility(h), v)
    finally:
        h.destroy()


def test_select_after_queued_frames(plugin, oracle):
    cloud = B.random_gaussians_3d_seeded(40000, 11)
    cloud.position_visibility[:, :3] *= np.float32(0.1)
    view = B.headless_view(320, 200)
    h = plugin.add_cloud(cloud)
    try:
        s = B.CloudSettings(global_scale=0.25, binning_rounds=False)
        for _ in range(4):
            plugin.render_view(h, s, view, asynchronous=True)
        mask = check_select(plugin, h, cloud.position_visibility, 0.08, 3)
        assert plugin.sync()                                     # nothing left queued
        check_frames(plugin, oracle, h, cloud, mask.astype(np.float32), view, "f32")
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
        mask = check_select(plugin, h, cloud.position_visibility, 0.08, 3)
        assert other.sync()
        img = other.render_view(h, s, view)
        til = oracle_frame(oracle, other, h, cloud, mask.astype(np.float32), s, view, "f32")
        assert np.abs(img - til["image"]).max() <= PIXEL_TOL
        plugin.set_visibility(h, np.ones(len(cloud), np.float32))
        other.render_view(h, s, view, asynchronous=True)
        plugin.invert_selection(h)
        assert other.sync()
        assert not plugin.visibility(h).any()
    finally:
        h.destroy()
        other.destroy()


def test_debug_hooks_not_ready_after_select_then_next_frame_matches(plugin, oracle):
    cloud = B.random_gaussians_3d_seeded(20000, 13)
    view = B.headless_view(320, 200)
    h = plugin.add_cloud(cloud)
    try:
        s = B.CloudSettings(global_scale=0.25, binning_rounds=False, draw_mode=B.DrawMode.Selected)
        plugin.render_view(h, s, view)
        plugin.frame_stats()
        plugin.select_sparse(h, B.SparseSelect(1.5, 4))
        for hook in (plugin.frame_stats, plugin.sorted_entries, plugin.tile_ranges, plugin.stage_times_us):
            with pytest.raises(abi.BgsError) as e:
                hook()
            assert e.value.status == abi.BGS_NOT_READY
        assert plugin.frame_device_ptr == 0
        vis = plugin.visibility(h)
        plugin.render_view(h, s, view)
        oc = B.PlanarGaussian3d(cloud.position_visibility.copy(), cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity)
        oc.position_visibility[:, 3] = vis
        u = plugin.cloud_uniform(s, None, h.aabb)
        keys = oracle.keygen(oc.position_visibility, view.to_abi(), u, 32)
        sk, si = oracle.radix_sort(keys, 32)
        got = plugin.sorted_entries()
        assert np.array_equal(got[:, 0], sk) and np.array_equal(got[:, 1], si)
        til = oracle.render_tiles(oc, view.to_abi(), u, s.to_abi())
        assert np.array_equal(plugin.tile_ranges(), til["tile_ranges"])
        assert np.array_equal(plugin.tile_entries(), til["tile_entries"])
    finally:
        h.destroy()


def test_errors(plugin):
    cloud = B.random_gaussians_3d_seeded(100, 0)
    h = plugin.add_cloud(cloud)
    lib, ctx = plugin._lib, plugin._ctx
    try:
        for r in (float("nan"), float("inf"), float("-inf"), -0.5):
            with pytest.raises(abi.BgsError) as e:
                plugin.select_sparse(h, B.SparseSelect(r, 3))
            assert e.value.status == abi.BGS_EINVAL
        assert np.all(plugin.visibility(h) == 1.0)             # a refused call changed nothing
        buf = np.zeros(100, np.float32)
        sel = C.c_uint32()
        assert lib.bgs_cloud_select_sparse(None, h._h, 0.1, 3, C.byref(sel)) == abi.BGS_EINVAL
        assert lib.bgs_cloud_select_sparse(ctx, None, 0.1, 3, C.byref(sel)) == abi.BGS_EINVAL
        assert lib.bgs_cloud_select_sparse(ctx, h._h, 0.1, 3, None) == abi.BGS_OK   # out_selected may be NULL
        for fn in (lib.bgs_cloud_visibility_get, lib.bgs_cloud_visibility_set):
            assert fn(None, h._h, buf.ctypes.data_as(C.c_void_p)) == abi.BGS_EINVAL
            assert fn(ctx, None, buf.ctypes.data_as(C.c_void_p)) == abi.BGS_EINVAL
            assert fn(ctx, h._h, None) == abi.BGS_EINVAL
    finally:
        h.destroy()


def test_cloud_on_another_device_is_refused():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    p0, p1 = B.GaussianSplattingPlugin(0), B.GaussianSplattingPlugin(1)
    h = p1.add_cloud(B.random_gaussians_3d_seeded(100, 0))
    try:
        for call in (lambda: p0.select_sparse(h), lambda: p0.visibility(h), lambda: p0.set_visibility(h, np.zeros(100))):
            with pytest.raises(abi.BgsError) as e:
                call()
            assert e.value.status == abi.BGS_EINVAL
    finally:
        h.destroy()
        p0.destroy()
        p1.destroy()
