"""GPU parity tests proper: the CUDA path, called through the C ABI (ctypes -> libbgs.so), against
the CPU oracle on the same seeded inputs.  Bar (BASELINE.json north_star): radix order and tile
ranges BIT-EXACT; per-pixel RGBA within 1e-3 L-inf (f32 accumulators).  Full-size configurations are
covered through size-independent properties (sortedness, permutation, range partition, idempotence,
compaction == sort-all)."""
import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import blend_cases as BC
import project_cases as PC

pytestmark = pytest.mark.gpu

PIXEL_TOL = 1e-3   # north_star: per-pixel RGBA within 1e-3 L-inf (f32)


@pytest.fixture(scope="module")
def plugin():
    p = B.GaussianSplattingPlugin(0)
    yield p
    p.destroy()


def _uniform(s):
    return B.GaussianSplattingPlugin.cloud_uniform(s)


def render_frame(plugin, h, settings, view, asynchronous=False, out=None):
    """One rgba32f frame.  `asynchronous`: enqueue it (BGS_FLAG_ASYNC), then `sync()`; a frame whose pair list outgrew
    the buffer is rendered again, as the API asks."""
    if not asynchronous:
        return plugin.render_view(h, settings, view, fmt="rgba32f", out=out)
    if out is None:
        out = np.empty((view.height, view.width, 4), np.float32)
    for _ in range(3):
        plugin.render_view(h, settings, view, fmt="rgba32f", out=out, asynchronous=True)
        if plugin.sync():
            return out
    raise AssertionError("a queued frame kept outgrowing the pair buffer")


def check_against_oracle(plugin, oracle, cloud, settings, view, f16=False, pixel_tol=PIXEL_TOL, ref_mode_too=False, cov=False,
                         asynchronous=False):
    h = plugin.add_cloud(cloud, f16=f16, precompute_covariance=cov)
    try:
        img = render_frame(plugin, h, settings, view, asynchronous)
        oc = cloud.rounded_to_f16() if f16 else cloud
        if cov:      # row f3: the oracle reads the decoded Covariance3dOpacityPacked128 from the plane slots it occupies
            oc = cloud.precomputed_covariance().rounded_to_f16()
        s_abi = settings.to_abi()
        s_abi.reserved = 1 if cov else 0
        u = plugin.cloud_uniform(settings, None, h.aabb)
        bits = int(settings.radix_sort_depth_bits)
        keys = oracle.keygen(oc.position_visibility, view.to_abi(), u, bits)
        sk, si = oracle.radix_sort(keys, bits)
        got = plugin.sorted_entries()
        assert np.array_equal(got[:, 0], sk), "sorted keys differ (must be bit-exact)"
        assert np.array_equal(got[:, 1], si), "sort permutation differs (must be bit-exact)"
        til = oracle.render_tiles(oc, view.to_abi(), u, s_abi)
        fs = plugin.frame_stats()
        assert fs.n_visible == til["n_vis"] and fs.n_pairs == til["n_pairs"]
        assert np.array_equal(plugin.tile_ranges(), til["tile_ranges"]), "tile ranges differ (must be bit-exact)"
        assert np.array_equal(plugin.tile_entries(), til["tile_entries"]), "per-tile slices differ"
        rec, ids = plugin.projected()
        assert np.array_equal(ids, til["rank_to_id"])
        orec = oracle.project(oc, view.to_abi(), u, s_abi, til["rank_to_id"])
        drawn = orec["xlo"] <= orec["xhi"]
        if settings.aabb and settings.gaussian_mode == B.GaussianMode.Gaussian3d:
            # USE_AABB record: centre, conic x/y/z, quad half-side
            geo = np.stack([orec["cx"], orec["cy"], orec["extra"][:, 0], orec["extra"][:, 1], orec["extra"][:, 2],
                            orec["extra"][:, 3]], 1)
        else:
            geo = np.stack([orec[k] for k in ("cx", "cy", "ux", "uy", "vx", "vy")], 1)
        # (bit-exact with the sign of zero counted; NaN as a class: its payload is not part of the result)
        assert PC.bits_agree(rec[drawn, :6], geo[drawn]).all(), "projected geometry not bit-exact"
        bb = rec[:, 6:8].view(np.uint32)
        assert np.array_equal(bb[drawn, 0], (orec["xlo"][drawn].astype(np.uint32) | (orec["xhi"][drawn].astype(np.uint32) << 16)))
        assert np.array_equal(bb[drawn, 1], (orec["ylo"][drawn].astype(np.uint32) | (orec["yhi"][drawn].astype(np.uint32) << 16)))
        assert np.all((bb[~drawn, 0] & 0xFFFF) > (bb[~drawn, 0] >> 16))      # empty bbox where the oracle's is
        dc = 1e-4                       # (Depth colours come from the frame pass, tests/test_gpu_project.py restates them)
        if drawn.any() and settings.rasterize_mode != B.RasterizeMode.Depth:   # orc_project leaves Depth colours to the frame pass
            col = np.stack([orec[k] for k in ("r", "g", "b")], 1)[drawn]
            assert PC.bits_agree(rec[drawn, 11], orec["op"][drawn]).all(), "opacity differs"
            if settings.rasterize_mode == B.RasterizeMode.Color:
                # the derived per-record bound of the SH colour path (rsqrt.approx, fma accumulation, __powf)
                bound = PC.colour_bound(oc, view, None, int(settings.color_space), ids[drawn])
                lit = (settings.draw_mode == B.DrawMode.HighlightSelected) & (oc.position_visibility[ids[drawn], 3] > 0.5)
                bound[lit] = 0.0
            else:                       # Normal / Position: the same IEEE operations on both sides
                bound = np.full(col.shape, 4 * PC.U) * np.maximum(1.0, np.abs(col))
            assert PC.colours_agree(rec[drawn, 8:11], col, bound).all(), "record colour outside its bound"
            with np.errstate(invalid="ignore"):
                diff = np.abs(rec[drawn, 8:11].astype(np.float64) - col)
            dc = float(np.max(np.where(np.isfinite(diff), diff, 0.0), initial=0.0))   # the measured record colour error
        err = float(np.abs(img - til["image"]).max())
        assert err <= pixel_tol, f"pixel L-inf {err}"
        # per pixel: within the derived error bound of the float64 evaluation of the same walk (blend_cases.blend_bounds)
        trace = oracle.blend_trace(oc, view.to_abi(), u, s_abi)
        bound, _ = BC.frame_bounds(trace, bool(settings.aabb), "opaque", dc)
        want = BC.expected_frame(trace, "opaque")

        def check_bound(frame, which):
            over = np.abs(frame.astype(np.float64) - want) - bound
            if over.max() > 0:
                y, x, c = np.unravel_index(int(over.argmax()), over.shape)
                raise AssertionError(f"{which}: pixel (x={x}, y={y}) channel {c} exceeds its error bound {bound[y, x, c]:.3g} "
                                     f"by {over[y, x, c]:.3g}")

        check_bound(img, "first frame")
        if ref_mode_too:
            # the reference's own semantics (instanced quads blended back-to-front, no tiles, no early-out), directly
            ref = oracle.render_ref(oc, view.to_abi(), u, s_abi)
            err_ref = float(np.abs(img - ref).max())
            assert err_ref <= pixel_tol, f"pixel L-inf {err_ref} vs the oracle's ref_mode"
        # the second frame picks kernel variants from the first frame's counts (sort tile size, raster variant)
        img2 = render_frame(plugin, h, settings, view, asynchronous)
        err2 = float(np.abs(img2 - til["image"]).max())
        assert err2 <= pixel_tol, f"pixel L-inf {err2} on the hinted frame"
        check_bound(img2, "hinted frame")     # (raster2_kernel's frame where large_footprint_raster holds)
        if plugin.frame_stats().rounds == 1:   # (a multi-round frame keeps only its last round's ranges)
            assert np.array_equal(plugin.tile_ranges(), til["tile_ranges"])
        return img, til
    finally:
        h.destroy()


CASES = [
    # n, w, h, scale, f16, bits, sort_all
    (1000, 256, 256, 1.0, False, 32, False),      # config C1
    (1000, 256, 256, 1.0, True, 32, False),
    (20000, 320, 200, 0.25, False, 32, False),
    (20000, 320, 200, 0.25, False, 32, True),
    (60000, 640, 360, 0.1, True, 32, False),
    (60000, 333, 177, 0.1, False, 24, False),     # viewport not a multiple of 16; 3-pass keys
    (60000, 333, 177, 0.1, False, 16, False),     # 2-pass keys (close depths collapse: stability matters)
    (60000, 640, 360, 0.05, True, 16, True),
    (8191, 64, 64, 0.5, False, 32, False),        # ragged tile counts everywhere
    (4097, 17, 9, 0.5, False, 32, True),          # tiny viewport
]


@pytest.mark.parametrize("n,w,h,scale,f16,bits,sort_all", CASES)
def test_parity_vs_oracle(plugin, oracle, n, w, h, scale, f16, bits, sort_all):
    cloud = B.random_gaussians_3d_seeded(n, n % 7)
    s = B.CloudSettings(global_scale=scale, radix_sort_depth_bits=B.RadixSortDepthBits(bits), sort_all=sort_all)
    check_against_oracle(plugin, oracle, cloud, s, B.headless_view(w, h), f16=f16)


def test_parity_settings_variants(plugin, oracle):
    cloud = B.random_gaussians_3d_seeded(15000, 11)
    view = B.orbit_view(3, 8, 400, 240)
    for kw in (dict(opacity_adaptive_radius=False), dict(global_opacity=1.8), dict(color_space=B.GaussianColorSpace.LinRec709Display),
               dict(rasterize_mode=B.RasterizeMode.Normal), dict(draw_mode=B.DrawMode.HighlightSelected),
               dict(rasterize_mode=B.RasterizeMode.Depth), dict(rasterize_mode=B.RasterizeMode.Depth, sort_all=True),
               dict(rasterize_mode=B.RasterizeMode.Depth, gaussian_mode=B.GaussianMode.Gaussian2d, aabb=True),
               dict(rasterize_mode=B.RasterizeMode.Normal, gaussian_mode=B.GaussianMode.Gaussian2d),
               dict(rasterize_mode=B.RasterizeMode.Position), dict(rasterize_mode=B.RasterizeMode.Position, sort_all=True)):
        s = B.CloudSettings(global_scale=0.2, **kw)
        check_against_oracle(plugin, oracle, cloud, s, view)


@pytest.mark.parametrize("gm,aabb,f16", [(B.GaussianMode.Gaussian3d, True, False), (B.GaussianMode.Gaussian2d, True, False),
                                         (B.GaussianMode.Gaussian2d, False, False), (B.GaussianMode.Gaussian2d, True, True)])
def test_parity_aabb_and_2dgs(plugin, oracle, gm, aabb, f16):
    """Rows a8 (2DGS surfels, gaussian_2d.wgsl:49-156) and the USE_AABB conic variant (gaussian.wgsl:459-471)."""
    cloud = B.random_gaussians_3d_seeded(25000, 13)
    for scale, view in ((0.25, B.headless_view(320, 200)), (0.08, B.orbit_view(2, 8, 417, 233))):
        s = B.CloudSettings(global_scale=scale, gaussian_mode=gm, aabb=aabb)
        check_against_oracle(plugin, oracle, cloud, s, view, f16=f16)


def test_parity_model_transform_and_draw_selected(plugin, oracle):
    cloud = B.random_gaussians_3d_seeded(12000, 5)
    cloud.position_visibility[::3, 3] = 0.0          # a third of the cloud is "unselected"
    m = np.eye(4, dtype=np.float32)
    a = 0.7
    m[:3, :3] = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]], np.float32) * np.float32(1.3)
    m[:3, 3] = [0.5, -0.25, 1.0]
    view = B.headless_view(320, 180)
    s = B.CloudSettings(global_scale=0.15, draw_mode=B.DrawMode.Selected)
    h = plugin.add_cloud(cloud)
    try:
        img = plugin.render_view(h, s, view, transform=B.CloudTransform(m))
        u = plugin.cloud_uniform(s, B.CloudTransform(m))
        til = oracle.render_tiles(cloud, view.to_abi(), u, s.to_abi())
        assert np.array_equal(plugin.tile_ranges(), til["tile_ranges"])
        assert np.abs(img - til["image"]).max() <= PIXEL_TOL
        keys = oracle.keygen(cloud.position_visibility, view.to_abi(), u, 32)
        sk, si = oracle.radix_sort(keys, 32)
        got = plugin.sorted_entries()
        assert np.array_equal(got[:, 0], sk) and np.array_equal(got[:, 1], si)
    finally:
        h.destroy()


def test_edge_cases(plugin, oracle):
    view = B.headless_view(96, 64)
    s = B.CloudSettings(global_scale=0.5)
    # a single gaussian
    one = B.PlanarGaussian3d(np.array([[0, 1.5, 0, 1]], np.float32), np.full((1, 48), 0.3, np.float32),
                             np.array([[0.9, 0.1, 0.2, 0.3]], np.float32), np.array([[0.5, 0.2, 0.3, 0.7]], np.float32))
    check_against_oracle(plugin, oracle, one, s, view)
    # every gaussian culled (behind the camera): black frame, empty ranges
    cloud = B.random_gaussians_3d_seeded(5000, 2)
    cloud.position_visibility[:, 2] = np.abs(cloud.position_visibility[:, 2]) + 6.0
    img, til = check_against_oracle(plugin, oracle, cloud, s, view)
    assert til["n_vis"] == 0 and til["n_pairs"] == 0 and np.all(img[..., :3] == 0) and np.all(img[..., 3] == 1)
    # degenerate inputs: zero opacity, zero scale, NaN position, identity rotation (NaN eigenvector quirk)
    deg = B.random_gaussians_3d_seeded(3000, 4)
    deg.scale_opacity[::5, 3] = 0.0
    deg.scale_opacity[1::5, :3] = 0.0
    deg.position_visibility[2::50, 0] = np.nan
    deg.rotation[3::5] = [1, 0, 0, 0]
    deg.scale_opacity[3::5, :3] = 0.3
    check_against_oracle(plugin, oracle, deg, s, view)


ROUND_CASES = [
    # n, w, h, scale, f16, settings
    (30000, 512, 384, 1.0, False, {}),                                      # every tile saturates early
    (60000, 333, 177, 0.3, True, {}),
    (30000, 512, 384, 0.05, False, {}),                                     # nothing saturates: all rounds emit
    (2000, 256, 256, 1.0, False, dict(global_opacity=0.05)),
    (20000, 400, 240, 0.6, False, dict(rasterize_mode=B.RasterizeMode.Depth)),
    (20000, 400, 240, 0.6, False, dict(rasterize_mode=B.RasterizeMode.Normal, sort_all=True)),
    (20000, 400, 240, 0.6, False, dict(gaussian_mode=B.GaussianMode.Gaussian2d)),
    (37, 96, 64, 1.0, False, {}),                                           # rounds with empty rank ranges
]


@pytest.mark.parametrize("n,w,h,scale,f16,kw", ROUND_CASES)
def test_binning_rounds_bit_identical(plugin, oracle, n, w, h, scale, f16, kw):
    """BGS_FLAG_CHUNKS: binning / tile sort / blend in front-to-back rank rounds that stop emitting pairs once every
    tile has saturated must give the one-round frame bit for bit (and so the oracle's within the pixel tolerance)."""
    cloud = B.random_gaussians_3d_seeded(n, 5)
    view = B.headless_view(w, h)
    hnd = plugin.add_cloud(cloud, f16=f16)
    try:
        one_s = B.CloudSettings(global_scale=scale, binning_rounds=False, **kw)
        many_s = B.CloudSettings(global_scale=scale, binning_rounds=True, **kw)
        for fmt in ("rgba32f", "rgba16f", "rgba8_srgb"):
            one = plugin.render_view(hnd, one_s, view, fmt=fmt)
            fs1 = plugin.frame_stats()
            pairs1, rounds1 = fs1.n_pairs, fs1.rounds
            many = plugin.render_view(hnd, many_s, view, fmt=fmt)
            fs2 = plugin.frame_stats()
            assert rounds1 == 1 and fs2.rounds > 1
            assert fs2.n_visible == fs1.n_visible and fs2.n_pairs <= pairs1
            assert np.array_equal(one.view(np.uint8), many.view(np.uint8)), fmt
            if fs2.tiles_saturated < fs2.tiles_x * fs2.tiles_y:
                assert fs2.n_pairs == pairs1          # some tile alive to the end: every pair was emitted
            many2 = plugin.render_view(hnd, many_s, view, fmt=fmt)      # hinted (per-round sort tile sizes)
            assert np.array_equal(one.view(np.uint8), many2.view(np.uint8)), fmt
        with pytest.raises(RuntimeError):
            plugin.tile_ranges()                      # the tile hooks need a one-round frame
        oc = cloud.rounded_to_f16() if f16 else cloud
        til = oracle.render_tiles(oc, view.to_abi(), _uniform(many_s), many_s.to_abi())
        img = plugin.render_view(hnd, many_s, view, fmt="rgba32f")
        assert float(np.abs(img - til["image"]).max()) <= PIXEL_TOL
    finally:
        hnd.destroy()


def test_binning_rounds_saturation_and_async(plugin):
    """A heavy scene saturates: later rounds emit nothing (fewer pairs than one round), also through async frames
    and through a pair buffer that has to grow mid-way."""
    cloud = B.random_gaussians_3d_seeded(200000, 8)
    view = B.headless_view(640, 360)
    p2 = B.GaussianSplattingPlugin(0)
    try:
        hnd = p2.add_cloud(cloud)
        one_s = B.CloudSettings(global_scale=1.0, binning_rounds=False)
        many_s = B.CloudSettings(global_scale=1.0, binning_rounds=True)
        out = np.empty((360, 640, 4), np.float32)
        p2.render_view(hnd, many_s, view, fmt="rgba32f", out=out, asynchronous=True)   # first frame: buffer too small
        if not p2.sync():
            p2.render_view(hnd, many_s, view, fmt="rgba32f", out=out, asynchronous=True)
            if not p2.sync():
                p2.render_view(hnd, many_s, view, fmt="rgba32f", out=out, asynchronous=True)
                assert p2.sync()
        fs = p2.frame_stats()
        pairs_rounds, sat = fs.n_pairs, fs.tiles_saturated
        assert fs.rounds > 1 and sat == fs.tiles_x * fs.tiles_y
        ref = p2.render_view(hnd, one_s, view, fmt="rgba32f")
        assert np.array_equal(out, ref)
        assert pairs_rounds < p2.frame_stats().n_pairs // 2
        hnd.destroy()
    finally:
        p2.destroy()


@pytest.mark.parametrize("with_model", [False, True])
def test_frustum_boundary_visibility_bit_exact(plugin, oracle, with_model):
    """Key-gen decides visibility with one approximate reciprocal and falls back to the exact IEEE divisions near the
    frustum bounds (|ndc.x|, |ndc.y| = 1.1, ndc.z = 0 / 1): gaussians placed within a few ulp of every bound, on both
    sides, must be classified exactly like the oracle's divisions do (transform.wgsl:5-14)."""
    view = B.orbit_view(1, 8, 320, 200)
    VP = view.clip_from_world.astype(np.float64)          # row-major (row, col)
    rng = np.random.default_rng(3)
    m = np.eye(4, dtype=np.float32)
    if with_model:
        m[:3, :3] = np.array([[0.8, 0.1, 0.0], [-0.1, 0.9, 0.2], [0.05, -0.2, 1.1]], np.float32)
        m[:3, 3] = [0.3, -0.2, 0.5]
    Minv = np.linalg.inv(m.astype(np.float64))
    pts = []
    VPinv = np.linalg.inv(VP)
    for _ in range(6000):
        # an interior point of the frustum in NDC with ONE coordinate put on its bound +- a few ulp, unprojected
        # (f64) and rounded to f32: the rounding alone scatters the points over both sides of the bound
        nd = np.array([rng.uniform(-0.9, 0.9), rng.uniform(-0.9, 0.9), 0.1 / rng.uniform(0.5, 30.0), 1.0])
        row = int(rng.integers(0, 3))
        t = [1.1, -1.1][int(rng.integers(0, 2))] if row < 2 else 1.0
        nd[row] = t * (1.0 + float(rng.integers(-6, 7)) * 2.0 ** -23)
        w = VPinv @ nd
        pts.append((Minv @ (w / w[3]))[:3])
    pts = np.asarray(pts, np.float32)
    pts = pts[np.isfinite(pts).all(1) & (np.abs(pts).max(1) < 1e4)]
    n = len(pts)
    cloud = B.random_gaussians_3d_seeded(n, 1)
    cloud.position_visibility[:, :3] = pts
    s = B.CloudSettings(global_scale=0.05)
    tr = B.CloudTransform(m) if with_model else None
    h = plugin.add_cloud(cloud)
    try:
        plugin.render_view(h, s, view, transform=tr, to_host=False)
        u = plugin.cloud_uniform(s, tr)
        keys = oracle.keygen(cloud.position_visibility, view.to_abi(), u, 32)
        vis = keys != 0xFFFFFFFF
        assert 0.15 * n < vis.sum() < 0.85 * n, "the construction must straddle the bounds"
        sk, si = oracle.radix_sort(keys, 32)
        got = plugin.sorted_entries()
        assert plugin.frame_stats().n_visible == int(vis.sum())
        assert np.array_equal(got[:, 0], sk) and np.array_equal(got[:, 1], si)
    finally:
        h.destroy()


def test_output_formats_agree(plugin):
    cloud = B.random_gaussians_3d_seeded(30000, 9)
    view = B.headless_view(320, 192)
    s = B.CloudSettings(global_scale=0.3)
    h = plugin.add_cloud(cloud)
    try:
        f32 = plugin.render_view(h, s, view, fmt="rgba32f")
        f16 = plugin.render_view(h, s, view, fmt="rgba16f")
        u8 = plugin.render_view(h, s, view, fmt="rgba8_srgb")
        assert np.abs(f16.astype(np.float32) - f32).max() <= 4e-3 * max(1.0, np.abs(f32).max())
        c = np.clip(f32[..., :3], 0, 1)
        enc = np.where(c <= 0.0031308, 12.92 * c, 1.055 * np.power(c, 1 / 2.4) - 0.055) * 255
        assert np.abs(u8[..., :3].astype(np.float32) - enc).max() <= 0.51
        assert np.all(u8[..., 3] == 255)
    finally:
        h.destroy()


def test_f16_target_within_2_ulp_of_oracle(plugin, oracle):
    """north_star: per-pixel RGBA within 2 ULP (f16) on the Rgba16Float target (render/mod.rs:917-921)."""
    cloud = B.random_gaussians_3d_seeded(20000, 21)
    view = B.headless_view(256, 144)
    s = B.CloudSettings(global_scale=0.3)
    h = plugin.add_cloud(cloud)
    try:
        got = plugin.render_view(h, s, view, fmt="rgba16f")
    finally:
        h.destroy()
    want = oracle.render_tiles(cloud, view.to_abi(), plugin.cloud_uniform(s), s.to_abi())["image"].astype(np.float16)
    # distance in f16 ULPs: reinterpret as sign-magnitude integers
    def ordinal(a):
        b = a.view(np.int16).astype(np.int32)
        return np.where(b < 0, -(b & 0x7FFF), b)
    assert np.abs(ordinal(got) - ordinal(want)).max() <= 2


def test_not_ready_and_bad_arguments(plugin):
    import ctypes as C

    from bevy_gaussian_splatting_b200 import abi

    lib = abi.load()
    v = B.headless_view(64, 64).to_abi(); s = B.CloudSettings().to_abi(); u = plugin.cloud_uniform(B.CloudSettings())
    # cloud asset not ready -> the reference skips the frame (radix.rs:645-658)
    assert lib.bgs_render(plugin._ctx, None, C.byref(v), C.byref(u), C.byref(s), None, 2, 0) == abi.BGS_NOT_READY
    h = plugin.add_cloud(B.random_gaussians_3d_seeded(100, 0))
    s.radix_sort_depth_bits = 20
    assert lib.bgs_render(plugin._ctx, h._h, C.byref(v), C.byref(u), C.byref(s), None, 2, 0) == abi.BGS_EINVAL
    assert b"radix_sort_depth_bits" in lib.bgs_last_error(plugin._ctx)
    h.destroy()


@pytest.mark.parametrize("n,f16,scale", [(1_000_000, False, 0.02), (6_000_000, True, 0.02)])
def test_full_size_properties(plugin, n, f16, scale):
    """Configs C2 / C3 at BASELINE.json's sizes: properties the oracle-free way."""
    cloud = B.random_gaussians_3d_seeded(n, 0)
    view = B.headless_view(1920, 1080)
    h = plugin.add_cloud(cloud, f16=f16)
    try:
        s = B.CloudSettings(global_scale=scale)
        img = plugin.render_view(h, s, view, fmt="rgba32f")
        ent = plugin.sorted_entries()
        fs = plugin.frame_stats()
        nv = fs.n_visible
        # sortedness + stability + permutation
        k = ent[:, 0].astype(np.int64)
        assert np.all(np.diff(k) >= 0)
        ties = np.diff(k) == 0
        assert np.all(np.diff(ent[:, 1].astype(np.int64))[ties] > 0), "ties must keep ascending index (stable)"
        assert np.array_equal(np.sort(ent[:, 1]), np.arange(n, dtype=np.uint32))
        assert np.all(ent[nv:, 0] == 0xFFFFFFFF) and np.all(ent[:nv, 0] != 0xFFFFFFFF)
        # keys are the key formula of the positions (recomputed in numpy f32 for the visible head)
        p = cloud.position_visibility[ent[:nv, 1], :3]
        d = p - np.array([0, 1.5, 5], np.float32)
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]).astype(np.float32) + d[:, 2] * d[:, 2]
        assert np.array_equal(0xFFFFFFFF - d2.astype(np.float32).view(np.uint32), ent[:nv, 0])
        # tile ranges partition the pair list; slices ascend in rank
        rng_ = plugin.tile_ranges().astype(np.int64)
        assert int((rng_[:, 1] - rng_[:, 0]).sum()) == fs.n_pairs
        ne = rng_[rng_[:, 1] > rng_[:, 0]]
        assert np.all(ne[1:, 0] == ne[:-1, 1]) and ne[0, 0] == 0 and ne[-1, 1] == fs.n_pairs
        te = plugin.tile_entries().astype(np.int64)
        brk = np.zeros(len(te), bool); brk[ne[:, 0]] = True
        assert np.all((np.diff(te) > 0) | brk[1:])
        # idempotence, and stream-compaction mode == reference-literal sort-all mode
        img2 = plugin.render_view(h, s, view, fmt="rgba32f")
        assert np.array_equal(img, img2)
        s_all = B.CloudSettings(global_scale=scale, sort_all=True)
        img3 = plugin.render_view(h, s_all, view, fmt="rgba32f")
        assert np.array_equal(img, img3)
        assert np.array_equal(plugin.sorted_entries(), ent)
        assert np.isfinite(img).all() and img[..., :3].max() > 0.05
    finally:
        h.destroy()


def test_full_size_surfels_and_auto_binning_rounds(plugin):
    """Config C4 (2 M surfels, 2DGS + USE_AABB, colour / depth / normal frames) and config C2's raw generator scale
    (global_scale 1: ~650 tiles per visible splat), at full size, through size-independent properties: idempotence,
    compaction == sort-all, finite output; and the library switching to binning rounds BY ITSELF on the heavy scene
    (from the first frame's statistics) without changing a bit of the frame."""
    view = B.headless_view(1920, 1080)
    cloud = B.random_gaussians_3d_seeded(2_000_000, 4)
    h = plugin.add_cloud(cloud)
    try:
        for rm in (B.RasterizeMode.Color, B.RasterizeMode.Depth, B.RasterizeMode.Normal):
            s = B.CloudSettings(global_scale=0.02, gaussian_mode=B.GaussianMode.Gaussian2d, aabb=True, rasterize_mode=rm)
            img = plugin.render_view(h, s, view, fmt="rgba32f")
            fs = plugin.frame_stats()
            assert fs.rounds == 1 and fs.n_visible > 100_000 and fs.n_pairs >= fs.n_visible // 2
            assert np.isfinite(img).all() and img[..., :3].max() > 0.05 and np.all(img[..., 3] == 1.0)
            assert np.array_equal(img, plugin.render_view(h, s, view, fmt="rgba32f"))
            import dataclasses
            assert np.array_equal(img, plugin.render_view(h, dataclasses.replace(s, sort_all=True), view, fmt="rgba32f"))
    finally:
        h.destroy()
    cloud = B.random_gaussians_3d_seeded(1_000_000, 0)
    p2 = B.GaussianSplattingPlugin(0)              # fresh context: no footprint statistics yet
    try:
        h2 = p2.add_cloud(cloud)
        s = B.CloudSettings(global_scale=1.0)
        first = p2.render_view(h2, s, view, fmt="rgba8_srgb")
        fs1 = p2.frame_stats()
        pairs1, rounds1 = fs1.n_pairs, fs1.rounds
        second = p2.render_view(h2, s, view, fmt="rgba8_srgb")
        fs2 = p2.frame_stats()
        assert rounds1 == 1 and pairs1 > 50_000_000                      # one round: every (splat, tile) pair
        assert fs2.rounds > 1 and fs2.n_pairs < pairs1 // 4              # rounds: the frame saturates early
        assert fs2.tiles_saturated == fs2.tiles_x * fs2.tiles_y
        assert np.array_equal(first, second)
        third = p2.render_view(h2, B.CloudSettings(global_scale=1.0, binning_rounds=False), view, fmt="rgba8_srgb")
        assert p2.frame_stats().rounds == 1 and np.array_equal(first, third)
        h2.destroy()
    finally:
        p2.destroy()


def test_async_frames_and_deferred_overflow(plugin):
    """BGS_FLAG_ASYNC: frames queue back to back; bgs_sync completes them; a pair-list overflow is reported at
    sync time (BGS_NOT_READY), the buffer grows, and the re-rendered frame is exact."""
    cloud = B.random_gaussians_3d_seeded(40000, 3)
    view = B.headless_view(640, 360)
    h = plugin.add_cloud(cloud)
    try:
        s = B.CloudSettings(global_scale=0.05)
        ref = plugin.render_view(h, s, view, fmt="rgba32f")
        for _ in range(3):
            plugin.render_view(h, s, view, fmt="rgba32f", to_host=False, asynchronous=True)
        out = np.empty_like(ref)
        plugin.render_view(h, s, view, fmt="rgba32f", out=out, asynchronous=True)
        assert plugin.sync()
        assert np.array_equal(out, ref)
        assert plugin.frame_stats().n_visible > 0
        # a much heavier frame (huge splats -> far more (splat, tile) pairs than the buffer holds)
        big = B.CloudSettings(global_scale=3.0)
        ref_big = None
        p2 = B.GaussianSplattingPlugin(0)
        try:
            h2 = p2.add_cloud(cloud)
            p2.render_view(h2, s, view, fmt="rgba32f", to_host=False)              # sizes the pair buffer small
            p2.render_view(h2, big, view, fmt="rgba32f", to_host=False, asynchronous=True)
            ok = p2.sync()
            pairs_needed_more = not ok
            out2 = np.empty_like(ref)
            p2.render_view(h2, big, view, fmt="rgba32f", out=out2, asynchronous=True)
            assert p2.sync()
            ref_big = plugin.render_view(h, big, view, fmt="rgba32f")              # synchronous path grows internally
            assert np.array_equal(out2, ref_big)
            assert pairs_needed_more or p2.frame_stats().n_pairs <= (1 << 20)
            h2.destroy()
        finally:
            p2.destroy()
    finally:
        h.destroy()


def test_cpp_host_example_matches_python_host(plugin, tmp_path):
    """The C++ host mirror (include/bgs.hpp, examples/headless.cpp -- the counterpart of the reference's
    examples/headless.rs) drives the same C ABI: its frame must be byte-identical to the ctypes host's."""
    import os
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "examples", "headless")
    if not os.path.exists(exe):
        subprocess.run(["make", "-C", os.path.join(root, "examples")], check=True)
    n, w, h, scale = 50000, 640, 360, 0.2
    cloud_f, raw_f = str(tmp_path / "cloud.bin"), str(tmp_path / "frame.raw")
    out = subprocess.run([exe, str(n), str(w), str(h), str(scale), str(tmp_path / "0.ppm"), "--dump-cloud", cloud_f, "--raw", raw_f],
                         check=True, capture_output=True, text=True).stdout
    assert "rendered=1" in out
    buf = np.fromfile(cloud_f, np.uint8)
    assert int(buf[:8].view(np.uint64)[0]) == n
    f = buf[8:].view(np.float32)
    cloud = B.PlanarGaussian3d(f[: n * 4].reshape(n, 4), f[n * 4: n * 52].reshape(n, 48), f[n * 52: n * 56].reshape(n, 4),
                               f[n * 56: n * 60].reshape(n, 4))
    hnd = plugin.add_cloud(cloud)
    try:
        img = plugin.render_view(hnd, B.CloudSettings(global_scale=scale), B.headless_view(w, h), fmt="rgba8_srgb")
    finally:
        hnd.destroy()
    cpp = np.fromfile(raw_f, np.uint8).reshape(h, w, 4)
    assert np.array_equal(cpp, img)
    assert img[..., :3].max() > 16


def test_visibility_render_scene_on_gpu(plugin, oracle):
    """tests/visibility_render.rs:113-141,199-274 through the CUDA path: 9 red gaussians, 128x128, camera (0,0,5),
    global_opacity 2, adaptive radius off => >= 64 pixels with max(rgb) > 8 and a max channel > 32; a cloud whose
    gaussians are all deselected under DrawMode::Selected (the test's "hidden" phase) leaves <= 8 such pixels."""
    sh = np.zeros(48, np.float32); sh[0] = 6.0
    pos = [[x, y, z, 1.0] for x in (-0.35, 0.35) for y in (-0.35, 0.35) for z in (-0.35, 0.35)]
    pos.append(pos[0])
    n = len(pos)
    cloud = B.PlanarGaussian3d(np.array(pos, np.float32), np.tile(sh, (n, 1)), np.tile(np.array([1, 0, 0, 0], np.float32), (n, 1)),
                               np.tile(np.array([0.22, 0.22, 0.22, 0.85], np.float32), (n, 1)))
    view = B.perspective_view((0, 0, 5), (0, 0, 0), 128, 128)
    s = B.CloudSettings(global_opacity=2.0, global_scale=1.0, opacity_adaptive_radius=False)
    img32, _ = check_against_oracle(plugin, oracle, cloud, s, view)
    h = plugin.add_cloud(cloud)
    try:
        img8 = plugin.render_view(h, s, view, fmt="rgba8_srgb")
        assert int((img8[..., :3].max(axis=2) > 8).sum()) >= 64 and int(img8[..., :3].max()) > 32
        assert img8[..., 0].max() >= img8[..., 1].max()
    finally:
        h.destroy()
    hidden = B.PlanarGaussian3d(np.concatenate([cloud.position_visibility[:, :3], np.zeros((n, 1), np.float32)], 1),
                                cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity)
    h = plugin.add_cloud(hidden)
    try:
        img8 = plugin.render_view(h, B.CloudSettings(global_opacity=2.0, opacity_adaptive_radius=False, draw_mode=B.DrawMode.Selected),
                                  view, fmt="rgba8_srgb")
        assert int((img8[..., :3].max(axis=2) > 8).sum()) <= 8
    finally:
        h.destroy()


FULL_SIZE = [
    # BASELINE.json configs at their full sizes, CUDA vs the oracle (not CUDA vs itself)
    ("C2", 1_000_000, False, dict(global_scale=0.02)),
    ("C3", 6_000_000, True, dict(global_scale=0.02)),                                          # the bench.py configuration
    ("C4-colour", 2_000_000, False, dict(global_scale=0.02, gaussian_mode=B.GaussianMode.Gaussian2d, aabb=True)),
    ("C4-depth", 2_000_000, False, dict(global_scale=0.02, gaussian_mode=B.GaussianMode.Gaussian2d, aabb=True,
                                        rasterize_mode=B.RasterizeMode.Depth)),
    ("C4-normal", 2_000_000, False, dict(global_scale=0.02, gaussian_mode=B.GaussianMode.Gaussian2d, aabb=True,
                                         rasterize_mode=B.RasterizeMode.Normal)),
]


@pytest.mark.parametrize("name,n,f16,kw", FULL_SIZE, ids=[c[0] for c in FULL_SIZE])
def test_full_size_vs_oracle(plugin, oracle, name, n, f16, kw):
    """The benchmarked frame itself (and C2 / C4) against the oracle at 1920x1080: sorted (key, index) entries, tile
    ranges, per-tile slices and projected geometry bit-exact; pixels <= 1e-3 vs the oracle's tile_mode AND vs its
    ref_mode (the reference's back-to-front semantics) directly.  Covers the regimes only full sizes reach: 4096-entry
    sort tiles, key-gen ranges that do not fit shared memory, > 65535-row grids, the footprint queues of the binning."""
    cloud = B.random_gaussians_3d_seeded(n, 4 if name.startswith("C4") else 0)
    check_against_oracle(plugin, oracle, cloud, B.CloudSettings(**kw), B.headless_view(1920, 1080), f16=f16, ref_mode_too=True)


def test_compositing_over_target_and_premultiplied(plugin, oracle):
    """Row (b): the reference blends every visible cloud over whatever the view target holds, PREMULTIPLIED_ALPHA_BLENDING,
    one Transparent3d item per cloud (render/mod.rs:398-452, :944-948).  BGS_FLAG_BLEND_OVER_TARGET / _PREMULTIPLIED_OUT
    against the oracle's ref_mode run over the same initial target."""
    view = B.orbit_view(1, 8, 384, 216)
    far = B.random_gaussians_3d_seeded(9000, 31)
    near = B.random_gaussians_3d_seeded(7000, 32)
    near.position_visibility[:, :3] *= np.float32(0.5)          # a smaller cloud in front of / inside the first one
    s_far, s_near = B.CloudSettings(global_scale=0.3), B.CloudSettings(global_scale=0.2, global_opacity=0.8)
    h_far, h_near = plugin.add_cloud(far), plugin.add_cloud(near, f16=True)
    try:
        u_far, u_near = plugin.cloud_uniform(s_far, None, h_far.aabb), plugin.cloud_uniform(s_near, None, h_near.aabb)
        near16 = near.rounded_to_f16()
        # two clouds in one target, far cloud first
        base = plugin.render_view(h_far, s_far, view, fmt="rgba32f")
        both = plugin.render_view(h_near, s_near, view, fmt="rgba32f", blend_over=True)
        want_base = oracle.render_ref(far, view.to_abi(), u_far, s_far.to_abi())
        want_both = oracle.render_ref(near16, view.to_abi(), u_near, s_near.to_abi(), dst=want_base)
        assert np.abs(base - want_base).max() <= PIXEL_TOL
        assert np.abs(both - want_both).max() <= PIXEL_TOL
        assert np.abs(both - base).max() > 0.05 and np.all(both[..., 3] == 1.0)       # it did blend, alpha stays opaque
        # the layer alone, premultiplied: (C, 1 - T)
        layer = plugin.render_view(h_near, s_near, view, fmt="rgba32f", premultiplied=True)
        want_layer = oracle.render_ref(near16, view.to_abi(), u_near, s_near.to_abi(), dst=np.zeros_like(want_base))
        assert np.abs(layer - want_layer).max() <= PIXEL_TOL
        assert layer[..., 3].min() >= 0.0 and layer[..., 3].max() > 0.5 and layer[..., 3].max() <= 1.0
        # compositing the layer by hand over the first frame == the blend-over frame
        assert np.abs(layer[..., :3] + (1.0 - layer[..., 3:4]) * base[..., :3] - both[..., :3]).max() <= 2e-5
        # a scene behind the splats: blend over an arbitrary (non-black, translucent) target held by the context
        far_layer = oracle.render_ref(far, view.to_abi(), u_far, s_far.to_abi(), dst=np.zeros_like(want_base))

        def srgb_enc(c):
            c = np.clip(c, 0, 1)
            return np.where(c <= 0.0031308, 12.92 * c, 1.055 * np.power(c, 1 / 2.4) - 0.055)

        def srgb_dec(c):
            return np.where(c <= 0.04045, c / 12.92, np.power((c + 0.055) / 1.055, 2.4))

        for fmt in ("rgba16f", "rgba8_srgb"):
            held = plugin.render_view(h_far, s_far, view, fmt=fmt, premultiplied=True)       # target <- far layer (C, 1 - T)
            got = plugin.render_view(h_near, s_near, view, fmt=fmt, blend_over=True).astype(np.float32)
            if fmt == "rgba8_srgb":
                # an 8-bit sRGB target clamps and quantises what it holds: blend over exactly what it held
                assert np.abs(held[..., :3] / 255.0 - srgb_enc(far_layer[..., :3])).max() <= 1.01 / 255.0
                h8 = held.astype(np.float32) / 255.0
                dst = np.concatenate([srgb_dec(h8[..., :3]), h8[..., 3:4]], axis=2).astype(np.float32)
                want = oracle.render_ref(near16, view.to_abi(), u_near, s_near.to_abi(), dst=dst)
                want = np.concatenate([srgb_enc(want[..., :3]), np.clip(want[..., 3:4], 0, 1)], axis=2)
                assert np.abs(got / 255.0 - want).max() <= 1.01 / 255.0
            else:
                want = oracle.render_ref(near16, view.to_abi(), u_near, s_near.to_abi(), dst=held.astype(np.float32))
                assert np.abs(got - want).max() <= 4e-3 * max(1.0, np.abs(want).max())
        # binning rounds take the same output path
        rounds = plugin.render_view(h_near, B.CloudSettings(global_scale=0.2, global_opacity=0.8, binning_rounds=True), view,
                                    fmt="rgba32f", premultiplied=True)
        assert plugin.frame_stats().rounds > 1 and np.array_equal(rounds, layer)
    finally:
        h_far.destroy(); h_near.destroy()


@pytest.mark.parametrize("gm,aabb,n,scale", [(B.GaussianMode.Gaussian2d, True, 40000, 0.12), (B.GaussianMode.Gaussian3d, False, 30000, 0.2),
                                             (B.GaussianMode.Gaussian3d, True, 20000, 0.25)])
def test_aux_depth_normal_frames_in_one_pass(plugin, oracle, gm, aabb, n, scale):
    """Row f2 / config C4: bgs_render_aux delivers colour + depth + normal frames from ONE pass; each must be the frame the
    corresponding single-mode bgs_render produces (gaussian.wgsl:329-368, material/depth.wgsl:3-11) -- bit for bit -- and so
    match the oracle's three single-mode frames within the pixel tolerance."""
    import dataclasses

    cloud = B.random_gaussians_3d_seeded(n, 41)
    view = B.orbit_view(3, 8, 480, 270)
    s = B.CloudSettings(global_scale=scale, gaussian_mode=gm, aabb=aabb)
    h = plugin.add_cloud(cloud)
    try:
        colour, depth, normal = plugin.render_view_aux(h, s, view, fmt="rgba32f")
        for got, mode in ((colour, B.RasterizeMode.Color), (depth, B.RasterizeMode.Depth), (normal, B.RasterizeMode.Normal)):
            sm = dataclasses.replace(s, rasterize_mode=mode)
            single = plugin.render_view(h, sm, view, fmt="rgba32f")
            assert np.array_equal(got, single), mode
            want = oracle.render_tiles(cloud, view.to_abi(), plugin.cloud_uniform(sm, None, h.aabb), sm.to_abi())["image"]
            assert np.abs(got - want).max() <= PIXEL_TOL, mode
        assert np.abs(depth - colour).max() > 0.05 and np.abs(normal - colour).max() > 0.05
        c8, d8, n8 = plugin.render_view_aux(h, s, view, fmt="rgba8_srgb")
        assert np.array_equal(c8, plugin.render_view(h, s, view, fmt="rgba8_srgb"))
        assert np.array_equal(n8, plugin.render_view(h, dataclasses.replace(s, rasterize_mode=B.RasterizeMode.Normal), view, fmt="rgba8_srgb"))
    finally:
        h.destroy()


def test_parity_precomputed_covariance_plane(plugin, oracle):
    """Row f3: `Covariance3dOpacityPacked128` clouds (the reference's precompute_covariance_3d layout, f16.rs:131-170,
    planar.wgsl:133-152, gaussian_3d.wgsl:78-79): same bit-exact / 1e-3 bars as the other layouts."""
    cloud = B.random_gaussians_3d_seeded(30000, 19)
    cloud.scale_opacity[:, :3] *= np.float32(0.15)          # (the stored covariance ignores global_scale: scale the cloud itself)
    for view, kw in ((B.headless_view(480, 270), {}), (B.orbit_view(5, 8, 417, 233), dict(rasterize_mode=B.RasterizeMode.Depth)),
                     (B.orbit_view(2, 8, 320, 200), dict(aabb=True, global_scale=7.0))):      # global_scale must NOT matter
        check_against_oracle(plugin, oracle, cloud, B.CloudSettings(**kw), view, f16=True, cov=True)
    h = plugin.add_cloud(cloud, precompute_covariance=True)
    try:
        a = plugin.render_view(h, B.CloudSettings(), B.headless_view(320, 200))
        b = plugin.render_view(h, B.CloudSettings(global_scale=3.0), B.headless_view(320, 200))
        assert np.array_equal(a, b)
        for bad in (dict(rasterize_mode=B.RasterizeMode.Normal), dict(gaussian_mode=B.GaussianMode.Gaussian2d)):
            with pytest.raises(B.BgsError):
                plugin.render_view(h, B.CloudSettings(**bad), B.headless_view(320, 200))
    finally:
        h.destroy()


def test_cloud_files_through_the_cuda_path(plugin, oracle, tmp_path):
    """Row f1 end to end ("same .gcloud/.ply input" in the north star): a cloud written as `.ply` (INRIA layout, the reference's
    quirks on the way back in: sigmoid / exp-clamp / normalise / pad-32, io/ply.rs:23-132) and as `.gcloud` (FlexBuffers serde,
    io/gcloud/flexbuffers.rs:9-22) -> `load_cloud` (io/loader.rs:38-66) -> upload -> CUDA frame, against the oracle run on the
    loaded planes; and the C++ loader (include/bgs_io.hpp) must hand the GPU the identical cloud."""
    import os
    import subprocess

    from bevy_gaussian_splatting_b200 import io as bio

    src = B.random_gaussians_3d_seeded(20000, 77)
    src.rotation /= np.linalg.norm(src.rotation, axis=1, keepdims=True)
    src.scale_opacity[:, :3] = src.scale_opacity[:, :3] * np.float32(0.05) + np.float32(0.005)
    src.scale_opacity[:, 3] = np.clip(src.scale_opacity[:, 3], 0.02, 0.98)
    view = B.orbit_view(6, 8, 448, 252)
    s = B.CloudSettings()
    bio.write_ply_3d(tmp_path / "scene.ply", src)
    B.write_gcloud(tmp_path / "scene.gcloud", src)
    frames = {}
    for name in ("scene.ply", "scene.gcloud"):
        cloud = B.load_cloud(tmp_path / name)
        assert len(cloud) >= len(src)
        img, til = check_against_oracle(plugin, oracle, cloud, s, view)
        assert til["n_vis"] > 1000 and img[..., :3].max() > 0.05
        frames[name] = img
    # (the .gcloud round trip is lossless; the .ply one goes through logit / log and the reader's f_rest `i / 16` quirk, so the
    # two pictures differ in the view-dependent colour terms: both are checked against the oracle on THEIR loaded planes above)
    assert np.array_equal(B.load_cloud(tmp_path / "scene.gcloud").spherical_harmonic, src.spherical_harmonic)
    # C++ host loader -> the same planes -> the same frame, bit for bit
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.run(["make", "-C", os.path.join(root, "examples"), "-s", "cloud_tool"], check=True)
    for name in ("scene.ply", "scene.gcloud"):
        subprocess.run([os.path.join(root, "examples", "cloud_tool"), str(tmp_path / name), str(tmp_path / "planes.bin")], check=True, capture_output=True)
        raw = open(tmp_path / "planes.bin", "rb").read()
        n = int(np.frombuffer(raw, "<u8", 1)[0])
        f = np.frombuffer(raw, "<f4", n * 60, 8)
        cpp = B.PlanarGaussian3d(f[: n * 4].reshape(n, 4), f[n * 4: n * 52].reshape(n, 48), f[n * 52: n * 56].reshape(n, 4), f[n * 56:].reshape(n, 4))
        h = plugin.add_cloud(cpp)
        try:
            img = plugin.render_view(h, s, view, fmt="rgba32f")
        finally:
            h.destroy()
        if name.endswith(".gcloud"):
            assert np.array_equal(img, frames[name])
        else:       # (libm exp / sigmoid of the two hosts may differ in the last ulp)
            assert np.abs(img - frames[name]).max() <= 1e-3


def test_exported_frame_target_round_trip(plugin):
    """Row f4 (hand-back): the frame is rendered into an allocation exported as a POSIX fd (what Vulkan / wgpu-hal import with
    VK_KHR_external_memory_fd); importing that fd again -- the consumer's side, here in CUDA terms -- must show the rendered
    frame, byte for byte, with no copy in between."""
    import ctypes as C
    import os

    from bevy_gaussian_splatting_b200 import abi

    lib = abi.load()
    w, h = 512, 288
    nbytes = w * h * 4
    ptr, fd, alloc = C.c_void_p(), C.c_int(-1), C.c_size_t(0)
    assert lib.bgs_frame_export_create(0, nbytes, C.byref(ptr), C.byref(fd), C.byref(alloc)) == abi.BGS_OK
    assert ptr.value and fd.value >= 0 and alloc.value >= nbytes
    cloud = B.random_gaussians_3d_seeded(30000, 61)
    hd = plugin.add_cloud(cloud)
    view, s = B.headless_view(w, h), B.CloudSettings(global_scale=0.3)
    other = C.c_void_p()
    try:
        want = plugin.render_view(hd, s, view, fmt="rgba8_srgb")
        plugin.render_view_to_device(hd, s, view, ptr.value, fmt="rgba8_srgb")
        assert lib.bgs_frame_export_import(0, fd.value, alloc.value, C.byref(other)) == abi.BGS_OK
        assert other.value and other.value != ptr.value          # a second mapping of the same physical allocation
        got = np.empty(nbytes, np.uint8)
        cu = C.CDLL("libcuda.so.1")                                      # read the consumer's mapping with the driver API
        cu.cuMemcpyDtoH_v2.argtypes = [C.c_void_p, C.c_uint64, C.c_size_t]
        assert cu.cuMemcpyDtoH_v2(got.ctypes.data_as(C.c_void_p), C.c_uint64(other.value), nbytes) == 0
        assert np.array_equal(got.reshape(h, w, 4), want)
        assert want[..., :3].max() > 16
    finally:
        hd.destroy()
        if other.value:
            lib.bgs_frame_export_destroy(other)
        lib.bgs_frame_export_destroy(ptr)
        os.close(fd.value)


def test_overflow_of_an_earlier_queued_frame_is_reported(plugin):
    """ADVICE r1: with BGS_FLAG_ASYNC a pair-list overflow used to be noticed only on the LAST queued frame.  The library now
    keeps a sticky device-side maximum over every frame queued since the last sync: a heavy frame followed by a light one
    must still make `bgs_sync` report BGS_NOT_READY (and grow the buffer), after which the same sequence succeeds."""
    cloud = B.random_gaussians_3d_seeded(40000, 3)
    view = B.headless_view(640, 360)
    light, heavy = B.CloudSettings(global_scale=0.05), B.CloudSettings(global_scale=3.0)
    p2 = B.GaussianSplattingPlugin(0)
    try:
        h2 = p2.add_cloud(cloud)
        p2.render_view(h2, light, view, fmt="rgba32f", to_host=False)                       # sizes the pair buffer small
        small_pairs = p2.frame_stats().n_pairs
        out_heavy, out_light = np.empty((360, 640, 4), np.float32), np.empty((360, 640, 4), np.float32)
        p2.render_view(h2, heavy, view, fmt="rgba32f", out=out_heavy, asynchronous=True)    # overflows ...
        p2.render_view(h2, light, view, fmt="rgba32f", out=out_light, asynchronous=True)    # ... but is not the last frame
        ok = p2.sync()
        ref_heavy = plugin.add_cloud(cloud)
        try:
            want_heavy = plugin.render_view(ref_heavy, heavy, view, fmt="rgba32f")
            needs_more = plugin.frame_stats().n_pairs > max(small_pairs, 1 << 20)
        finally:
            ref_heavy.destroy()
        assert needs_more, "the construction must overflow the first buffer"
        assert not ok, "an overflow of the earlier frame went unreported"
        p2.render_view(h2, heavy, view, fmt="rgba32f", out=out_heavy, asynchronous=True)
        p2.render_view(h2, light, view, fmt="rgba32f", out=out_light, asynchronous=True)
        assert p2.sync()
        assert np.array_equal(out_heavy, want_heavy)
        h2.destroy()
    finally:
        p2.destroy()


@pytest.mark.gpu
def test_copy_engine_gather_with_device_side_signalling(plugin):
    """Row e (copy-engine gather): frames pushed into a frame stack with bgs_push_frame_signal, the consumer's stream held by
    bgs_wait_frames until every slot's sequence word has arrived.  One process and one GPU here (the slots are written by the
    same device); the cross-process form runs in bench.py --gpus N (`gather_ce`)."""
    import ctypes as C

    import torch

    from bevy_gaussian_splatting_b200 import abi

    lib = abi.load()
    w, h, slots = 320, 200, 3
    nbytes = w * h * 4
    flags_off = (slots * nbytes + 255) & ~255
    base, handle = C.c_void_p(), (C.c_ubyte * 64)()
    assert lib.bgs_peer_buffer_create(0, flags_off + 4 * slots, C.byref(base), handle) == abi.BGS_OK
    flags = C.c_void_p(base.value + flags_off)
    cu = C.CDLL("libcuda.so.1")
    cu.cuMemcpyDtoH_v2.argtypes = [C.c_void_p, C.c_uint64, C.c_size_t]

    def read(ptr, n):
        got = np.empty(n, np.uint8)
        assert cu.cuMemcpyDtoH_v2(got.ctypes.data_as(C.c_void_p), C.c_uint64(ptr), n) == 0
        return got

    hd = plugin.add_cloud(B.random_gaussians_3d_seeded(20000, 7))
    s = B.CloudSettings(global_scale=0.3)
    consumer = torch.cuda.Stream()
    try:
        assert not read(flags.value, 4 * slots).any()                     # the allocation starts cleared
        wants = []
        for seq in (1, 2):
            for i in range(slots):
                view = B.perspective_view((4.0 * np.cos(i + seq), 1.5, 4.0 * np.sin(i + seq)), (0, 0, 0), w, h)
                wants.append(plugin.render_view(hd, s, view, fmt="rgba8_srgb"))
                plugin.render_view(hd, s, view, fmt="rgba8_srgb", to_host=False, asynchronous=True)
                st = lib.bgs_push_frame_signal(plugin._ctx, C.c_void_p(plugin.frame_device_ptr), base, i, nbytes, flags, seq)
                assert st == abi.BGS_OK
            assert lib.bgs_wait_frames(C.c_void_p(consumer.cuda_stream), flags, slots, seq) == abi.BGS_OK
            consumer.synchronize()                                        # returns only when all three words reached seq
            got = read(base.value, slots * nbytes).reshape(slots, h, w, 4)
            for i in range(slots):
                assert np.array_equal(got[i], wants[-slots + i]), (seq, i)
            assert np.array_equal(read(flags.value, 4 * slots).view(np.uint32), np.full(slots, seq, np.uint32))
        # the compare is a cyclic >=: waiting for an older sequence passes at once
        assert lib.bgs_wait_frames(C.c_void_p(consumer.cuda_stream), flags, slots, 1) == abi.BGS_OK
        consumer.synchronize()
        assert plugin.sync()
        assert lib.bgs_wait_frames(None, None, slots, 1) == abi.BGS_EINVAL
        assert lib.bgs_push_frame_signal(plugin._ctx, C.c_void_p(plugin.frame_device_ptr), base, 0, nbytes, None, 1) == abi.BGS_EINVAL
    finally:
        hd.destroy()
        lib.bgs_peer_buffer_release(base, 0)
