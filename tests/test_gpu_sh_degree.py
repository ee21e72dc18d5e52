"""Clouds stored at SH degree 0, 1 and 2 on the GPU (the _sh upload and download calls; the rule: include/bgs.h).

* Equivalence, bit for bit: in every layout (f32, f16, f16 covariance), geometry (3D OBB and AABB, 2DGS with and
  without USE_AABB) and 3D rasterize mode, a degree-d cloud renders exactly like the same cloud zero-padded to degree 3
  through the degree-3 upload -- the RGBA32F frame, the projected records, the sorted entries and the tile ranges.
* The oracle: degree-d Color frames (of the zero-padded cloud) within smoke()'s bound, tile ranges exact.
* Padding lanes: non-zero values there change no frame.
* Round trips and edits: downloads return the upload's bytes; subsets keep the degree and equal the host subset;
  interpolation equals the interpolate oracle at S_d lanes and refuses clouds of different degrees; selection, particle
  steps and visibility work; queued, depth-tested and aux frames at degree 0 equal the padded cloud's.
* Degree 3 through the _sh calls is the degree-3 upload; the downloads without _sh refuse degree < 3.
"""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import sh_degree_cases as SC
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import PlanarGaussian3dHandle
from interpolate_oracle import interpolate_oracle as IO

pytestmark = pytest.mark.gpu

RM, GM = B.RasterizeMode, B.GaussianMode
N = 4000
VIEW = B.headless_view(256, 192)
PREV = B.perspective_view((0.03, 1.48, 5.05), (0.03, 1.48, 4.05), 256, 192)
GEOMETRIES = {"obb": (GM.Gaussian3d, False), "aabb": (GM.Gaussian3d, True), "surfel": (GM.Gaussian2d, False),
              "surfel_aabb": (GM.Gaussian2d, True)}
MODES = [RM.Color, RM.Depth, RM.Normal, RM.Position, RM.Classification, RM.OpticalFlow]


@pytest.fixture(scope="module")
def plugin():
    p = B.GaussianSplattingPlugin(0)
    yield p
    p.destroy()


def add(plugin, cloud, layout):
    return plugin.add_cloud(cloud, f16=layout == "f16", precompute_covariance=layout == "cov")


_HANDLES = {}


@pytest.fixture(scope="module")
def pair(plugin):
    """(degree-d handle, handle of the same cloud zero-padded to degree 3), uploaded once per (d, layout)."""
    def get(d, layout):
        if (d, layout) not in _HANDLES:
            c = SC.labelled_cloud(N, 40 + d, d)
            _HANDLES[(d, layout)] = (add(plugin, c, layout), add(plugin, c.with_sh_degree(3), layout))
        return _HANDLES[(d, layout)]
    yield get
    for a, b in _HANDLES.values():
        a.destroy(); b.destroy()
    _HANDLES.clear()


def settings_for(geometry, mode):
    gm, aabb = GEOMETRIES[geometry]
    return B.CloudSettings(global_scale=0.25, gaussian_mode=gm, aabb=aabb, rasterize_mode=mode, num_classes=4,
                           binning_rounds=False)


def frame(plugin, h, s, **kw):
    """Everything a frame leaves readable: the RGBA32F frame and the debug hooks."""
    if s.rasterize_mode == RM.OpticalFlow:
        kw = dict(previous_view=PREV, delta_time=1.0 / 60.0, **kw)
    img = plugin.render_view(h, s, VIEW, fmt="rgba32f", **kw)
    rec, ids = plugin.projected()
    return {"frame": img.tobytes(), "records": rec.tobytes(), "ids": ids.tobytes(),
            "sorted": plugin.sorted_entries().tobytes(), "ranges": plugin.tile_ranges().tobytes()}


def assert_same(a, b):
    for k in a:
        assert a[k] == b[k], k


def _equivalence_params():
    out = []
    for d in SC.DEGREES:
        for layout in SC.LAYOUTS:
            for g in GEOMETRIES:
                for m in MODES:
                    if layout == "cov" and (GEOMETRIES[g][0] != GM.Gaussian3d or m == RM.Normal):
                        continue   # (the covariance layout holds no rotation: bgs_render refuses these)
                    out.append((d, layout, g, m))
    return out


@pytest.mark.parametrize("d,layout,geometry,mode", _equivalence_params())
def test_degree_d_renders_like_zero_padded_degree_3(plugin, pair, d, layout, geometry, mode):
    hd, h3 = pair(d, layout)
    assert hd.sh_degree == d and h3.sh_degree == 3
    s = settings_for(geometry, mode)
    a = frame(plugin, hd, s)
    assert plugin.frame_stats().n_visible > 100
    b = frame(plugin, h3, s)
    assert_same(a, b)


@pytest.mark.parametrize("d", SC.DEGREES)
@pytest.mark.parametrize("layout", ["f32", "f16"])
def test_degree_d_frames_match_the_oracle(plugin, oracle, d, layout):
    c = B.random_gaussians_3d_seeded(20000, 60 + d, sh_degree=d)
    h = add(plugin, c, layout)
    try:
        s = B.CloudSettings(global_scale=0.25, binning_rounds=False)
        img = plugin.render_view(h, s, VIEW, fmt="rgba32f")
        ref_cloud = (c.rounded_to_f16() if layout == "f16" else c).with_sh_degree(3)
        u = plugin.cloud_uniform(s, None, h.aabb)
        til = oracle.render_tiles(ref_cloud, VIEW.to_abi(), u, s.to_abi())
        assert np.array_equal(plugin.tile_ranges(), til["tile_ranges"])
        err = float(np.abs(img - til["image"]).max())
        assert err <= 1e-3, err
    finally:
        h.destroy()


@pytest.mark.parametrize("d", [0, 2])
@pytest.mark.parametrize("layout", SC.LAYOUTS)
@pytest.mark.parametrize("mode", [RM.Color, RM.Classification])
def test_padding_lanes_change_no_frame(plugin, d, layout, mode):
    c = SC.labelled_cloud(N, 70 + d, d)
    noisy = SC.with_padding_noise(c, 71)
    h0, h1 = add(plugin, c, layout), add(plugin, noisy, layout)
    try:
        for g in ("obb", "aabb"):
            s = settings_for(g, mode)
            assert_same(frame(plugin, h0, s), frame(plugin, h1, s))
    finally:
        h0.destroy(); h1.destroy()


def upload_planes(cloud, layout):
    if layout == "f32":
        return cloud.position_visibility, cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity
    src = cloud.precomputed_covariance() if layout == "cov" else cloud
    return (cloud.position_visibility,) + src.pack_f16()


def assert_planes_equal(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.shape == w.shape and np.array_equal(np.ascontiguousarray(g).view(np.uint32), np.ascontiguousarray(w).view(np.uint32))


@pytest.mark.parametrize("d", SC.DEGREES)
@pytest.mark.parametrize("layout", SC.LAYOUTS)
def test_download_returns_the_upload_and_subsets_keep_the_degree(plugin, d, layout):
    c = B.random_gaussians_3d_seeded((1 << 19) + 1000, 80 + d, sh_degree=d)   # more than one download chunk at every degree
    if d in (0, 2):
        c = SC.with_padding_noise(c, 81)
    c.position_visibility[:, 3] = (np.arange(len(c)) % 3 == 0).astype(np.float32)
    h = add(plugin, c, layout)
    try:
        assert_planes_equal(plugin.download_planes(h), upload_planes(c, layout))
        if layout == "f32":
            back = plugin.download(h)
            assert back.sh_degree == d
        # the downloads of degree 3 refuse the cloud
        lib = plugin._lib
        n = len(c)
        pos, sh48, r4, s4 = (np.empty((n, 4), np.float32), np.empty((n, 48), np.float32), np.empty((n, 4), np.float32),
                             np.empty((n, 4), np.float32))
        sh24 = np.empty((n, 24), np.uint32)
        if layout == "f32":
            st = lib.bgs_cloud_download_f32(plugin._ctx, h._h, *(a.ctypes.data for a in (pos, sh48, r4, s4)))
            st16 = lib.bgs_cloud_download_f16_sh(plugin._ctx, h._h, *(a.ctypes.data for a in (pos, sh24, r4)))
        else:
            st = lib.bgs_cloud_download_f16(plugin._ctx, h._h, *(a.ctypes.data for a in (pos, sh24, r4)))
            st16 = lib.bgs_cloud_download_f32_sh(plugin._ctx, h._h, *(a.ctypes.data for a in (pos, sh48, r4, s4)))
        assert st == abi.BGS_EINVAL and st16 == abi.BGS_EINVAL
        # subsets, both modes
        idx = np.random.default_rng(d).integers(0, n, 5000)
        for sub, want in ((plugin.subset(h, idx), c.subset(idx)),
                          (plugin.subset(h), c.subset(np.flatnonzero(~(c.position_visibility[:, 3] < 0.5))))):
            try:
                assert sub.sh_degree == d and sub.n == len(want)
                assert_planes_equal(plugin.download_planes(sub), upload_planes(want, layout))
            finally:
                sub.destroy()
    finally:
        h.destroy()


@pytest.mark.parametrize("d", SC.DEGREES)
@pytest.mark.parametrize("layout", SC.LAYOUTS)
def test_interpolate_matches_the_oracle_at_s_d_lanes(plugin, d, layout):
    n = 3000
    lc = SC.with_padding_noise(B.random_gaussians_3d_seeded(n, 90, sh_degree=d), 1) if d != 1 else \
        B.random_gaussians_3d_seeded(n, 90, sh_degree=d)
    rc = SC.with_padding_noise(B.random_gaussians_3d_seeded(n, 91, sh_degree=d), 2) if d != 1 else \
        B.random_gaussians_3d_seeded(n, 91, sh_degree=d)
    hl, hr = add(plugin, lc, layout), add(plugin, rc, layout)
    out = plugin.subset(hl, np.arange(n))
    try:
        s = B.CloudSettings(time=0.3, time_start=0.0, time_stop=1.0)
        plugin.interpolate(out, hl, hr, s)
        assert plugin.sync()
        got = plugin.download_planes(out)
        embed = SC.embed48 if layout == "f32" else SC.embed24
        lp, rp = list(upload_planes(lc, layout)), list(upload_planes(rc, layout))
        lp[1], rp[1] = embed(lp[1]), embed(rp[1])
        want = list(IO.interpolate(layout, lp, rp, IO.factor(0.3, 0.0, 1.0)))
        want[1] = want[1][:, :got[1].shape[1]]
        assert_planes_equal(got, want)
        # a degree mismatch is refused, nothing enqueued
        other = add(plugin, B.random_gaussians_3d_seeded(n, 92, sh_degree=(d + 1) % 4), layout)
        try:
            for trio in ((out, hl, other), (out, other, hr), (other, hl, hr)):
                st = plugin._lib.bgs_cloud_interpolate(plugin._ctx, trio[0]._h, trio[1]._h, trio[2]._h, C.c_float(0.3),
                                                       C.c_float(0.0), C.c_float(1.0))
                assert st == abi.BGS_EINVAL
        finally:
            other.destroy()
    finally:
        out.destroy(); hl.destroy(); hr.destroy()


@pytest.mark.parametrize("d", SC.DEGREES)
def test_select_particles_and_visibility_on_degree_d(plugin, d):
    c = B.random_gaussians_3d_seeded(20000, 100 + d, sh_degree=d)
    c.position_visibility[:, :3] *= np.float32(0.05)   # dense enough for SparseSelect to find neighbours
    hd, h3 = add(plugin, c, "f32"), add(plugin, c.with_sh_degree(3), "f32")
    try:
        q = B.SparseSelect(radius=0.05, neighbor_threshold=3)
        assert plugin.select_sparse(hd, q) == plugin.select_sparse(h3, q)
        assert np.array_equal(plugin.visibility(hd), plugin.visibility(h3))
        tri = np.array([[-0.5, -0.5, -0.5], [0.5, -0.5, -0.5], [0.0, 0.5, -0.5], [0.0, 0.0, 0.5]], np.float32)
        faces = np.array([[0, 1, 2], [0, 1, 3], [1, 2, 3], [0, 2, 3]], np.uint32)
        assert plugin.select_in_mesh(hd, tri, faces) == plugin.select_in_mesh(h3, tri, faces)
        assert np.array_equal(plugin.visibility(hd), plugin.visibility(h3))
        vis = (np.arange(len(c)) % 2).astype(np.float32)
        plugin.set_visibility(hd, vis); plugin.set_visibility(h3, vis)
        assert np.array_equal(plugin.visibility(hd), vis)
        from bevy_gaussian_splatting_b200.particles import random_particle_behaviors
        parts = plugin.add_particles(random_particle_behaviors(5000, 3))
        try:
            for _ in range(3):
                plugin.step_particles(hd, parts, 0.1)
            parts2 = plugin.add_particles(random_particle_behaviors(5000, 3))
            for _ in range(3):
                plugin.step_particles(h3, parts2, 0.1)
            assert plugin.sync()
            assert np.array_equal(plugin.positions(hd), plugin.positions(h3))
            s = B.CloudSettings(global_scale=0.25, draw_mode=B.DrawMode.Selected, binning_rounds=False)
            assert_same(frame(plugin, hd, s), frame(plugin, h3, s))
            s = dataclasses.replace(s, draw_mode=B.DrawMode.HighlightSelected)
            assert_same(frame(plugin, hd, s), frame(plugin, h3, s))
            parts2.destroy()
        finally:
            parts.destroy()
    finally:
        hd.destroy(); h3.destroy()


@pytest.mark.parametrize("layout", SC.LAYOUTS)
def test_queued_depth_tested_and_aux_frames_at_degree_0(plugin, pair, layout):
    import torch

    hd, h3 = pair(0, layout)
    s = B.CloudSettings(global_scale=0.25)
    # queued: three frames in flight, alternating the two clouds, then compared with their synchronous frames
    outs = [np.empty((VIEW.height, VIEW.width, 4), np.float32) for _ in range(4)]
    for i, o in enumerate(outs):
        plugin.render_view(hd if i % 2 == 0 else h3, s, VIEW, fmt="rgba32f", out=o, asynchronous=True)
    assert plugin.sync()
    assert outs[0].tobytes() == outs[1].tobytes() == outs[2].tobytes() == outs[3].tobytes()
    assert outs[0].tobytes() == plugin.render_view(hd, s, VIEW, fmt="rgba32f").tobytes()
    # depth-tested against a plane through the cloud
    z = torch.full((VIEW.height, VIEW.width), 0.01, dtype=torch.float32, device="cuda")   # hides splats past 10 units
    a = plugin.render_view(hd, s, VIEW, fmt="rgba32f", scene_depth=z)
    da = plugin.splat_depths()
    b = plugin.render_view(h3, s, VIEW, fmt="rgba32f", scene_depth=z)
    assert a.tobytes() == b.tobytes() and da.tobytes() == plugin.splat_depths().tobytes()
    assert a.tobytes() != outs[0].tobytes()   # the test hid something
    # colour, depth and normal in one pass (the covariance layout has no normal: refused for both)
    if layout != "cov":
        fa = plugin.render_view_aux(hd, s, VIEW)
        fb = plugin.render_view_aux(h3, s, VIEW)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(fa, fb))


@pytest.mark.parametrize("layout", SC.LAYOUTS)
def test_degree_3_through_the_sh_calls_is_the_degree_3_upload(plugin, layout):
    c = SC.labelled_cloud(N, 110, 3)
    h_sh = add(plugin, c, layout)   # the plugin uploads through the _sh calls
    lib, ctx = plugin._lib, plugin._ctx
    raw = C.c_void_p()
    planes = upload_planes(c, layout)
    ptrs = [a.ctypes.data for a in planes]
    if layout == "f32":
        st = lib.bgs_cloud_upload_f32(ctx, N, *ptrs, C.byref(raw))
    elif layout == "f16":
        st = lib.bgs_cloud_upload_f16(ctx, N, *ptrs, C.byref(raw))
    else:
        st = lib.bgs_cloud_upload_f16_cov(ctx, N, *ptrs, C.byref(raw))
    assert st == abi.BGS_OK
    h_old = PlanarGaussian3dHandle._adopt(plugin, raw, N, layout == "f16", layout == "cov")
    try:
        assert h_old.sh_degree == 3
        for g in ("obb", "aabb") + (("surfel",) if layout != "cov" else ()):
            for m in (RM.Color, RM.Classification):
                s = settings_for(g, m)
                assert_same(frame(plugin, h_sh, s), frame(plugin, h_old, s))
        assert_planes_equal(plugin.download_planes(h_sh), planes)
        # the downloads without _sh read the same bytes
        n = N
        pos = np.empty((n, 4), np.float32)
        if layout == "f32":
            sh, r4, s4 = np.empty((n, 48), np.float32), np.empty((n, 4), np.float32), np.empty((n, 4), np.float32)
            assert lib.bgs_cloud_download_f32(ctx, h_sh._h, *(a.ctypes.data for a in (pos, sh, r4, s4))) == abi.BGS_OK
            assert_planes_equal((pos, sh, r4, s4), planes)
        else:
            sh, r4 = np.empty((n, 24), np.uint32), np.empty((n, 4), np.uint32)
            assert lib.bgs_cloud_download_f16(ctx, h_sh._h, *(a.ctypes.data for a in (pos, sh, r4))) == abi.BGS_OK
            assert_planes_equal((pos, sh, r4), planes)
    finally:
        h_sh.destroy(); h_old.destroy()


def test_refusals(plugin):
    lib, ctx = plugin._lib, plugin._ctx
    c = B.random_gaussians_3d_seeded(64, 5)
    out = C.c_void_p()
    shp, rso = c.pack_f16()
    p = c.position_visibility.ctypes.data
    assert lib.bgs_cloud_upload_f32_sh(ctx, 64, 4, p, c.spherical_harmonic.ctypes.data, c.rotation.ctypes.data,
                                       c.scale_opacity.ctypes.data, C.byref(out)) == abi.BGS_EINVAL and not out.value
    assert lib.bgs_cloud_upload_f16_sh(ctx, 64, 4, p, shp.ctypes.data, rso.ctypes.data, C.byref(out)) == abi.BGS_EINVAL
    assert lib.bgs_cloud_upload_f16_cov_sh(ctx, 64, 99, p, shp.ctypes.data, rso.ctypes.data, C.byref(out)) == abi.BGS_EINVAL
    assert not out.value
    h = plugin.add_cloud(c)
    d = C.c_uint32(9)
    assert lib.bgs_cloud_sh_degree(h._h, None) == abi.BGS_EINVAL
    assert lib.bgs_cloud_sh_degree(h._h, C.byref(d)) == abi.BGS_OK and d.value == 3
    h.destroy()
    # 4D clouds: degree 3, and no _sh download
    c4 = B.random_gaussians_4d_seeded(64, 1)
    h4 = plugin.add_cloud(c4)
    try:
        assert lib.bgs_cloud_sh_degree(h4._h, C.byref(d)) == abi.BGS_OK and d.value == 3
        bufs = [np.empty((64, w), np.float32) for w in (4, 48, 4, 4)]
        assert lib.bgs_cloud_download_f32_sh(ctx, h4._h, *(a.ctypes.data for a in bufs)) == abi.BGS_EINVAL
        w = [np.empty((64, k), np.uint32) for k in (4, 24, 4)]
        assert lib.bgs_cloud_download_f16_sh(ctx, h4._h, *(a.ctypes.data for a in w)) == abi.BGS_EINVAL
    finally:
        h4.destroy()
