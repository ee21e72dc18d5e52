"""The bounding-box overlay (BGS_FLAG_VISUALIZE_BOUNDING_BOX, bgs_render_entities_ex's per-entity bit) on the H100.

With BGS_FLAG_PREMULTIPLIED_OUT and RGBA32F a pixel's alpha 1 - T is exactly 1.0f iff an edge blended there: a pixel
stops at T < 1e-4 and no other blend takes T below 1e-7, so 1 - T reaches 1.0f only through an edge's T = 0.  That makes
the edge mask of any frame observable bit for bit, and it is held to the entity oracle's (eo_frame_ex) for every blend
kind, with and without a depth buffer, queued and synchronous; the colour stays within 1e-3 of the oracle's."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

import bbox_cases as BX
import blend_cases as BC
import bevy_gaussian_splatting_b200 as B
import entity_cases as E
import scene4d_cases as S4
import scene_cases as SC
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import entity_settings
from entity_oracle import entity_oracle as EO

pytestmark = pytest.mark.gpu

PIXEL_TOL = 1e-3
BOX, PREMUL = abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX, abi.BGS_FLAG_PREMULTIPLIED_OUT
F32 = abi.BGS_FORMAT_RGBA32F


def _zd(depth, w):
    return None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * w)


def _depth(h, w, seed, scale=0.3):
    return torch.rand((h, w), generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda") * scale


def render(p, h, st, view, flags=0, depth=None):
    """One single-cloud frame in RGBA32F: bgs_render_4d for a 4D cloud, bgs_render_depth_test under a depth buffer,
    else bgs_render_ex."""
    w, hh = int(view.width), int(view.height)
    s = st.to_abi()
    s.flags |= flags
    u = p.cloud_uniform(st, None, h.aabb)
    out = np.empty((hh, w, 4), np.float32)
    zd = _zd(depth, w)
    if st.gaussian_mode == B.GaussianMode.Gaussian4d:
        rc = p._lib.bgs_render_4d(p._ctx, h._h, C.byref(view.to_abi()), C.byref(u), C.byref(s), None,
                                  None if zd is None else C.byref(zd), out.ctypes.data, F32, 0, C.c_float(st.time_start),
                                  C.c_float(st.time_stop))
    elif zd is not None:
        rc = p._lib.bgs_render_depth_test(p._ctx, h._h, C.byref(view.to_abi()), C.byref(u), C.byref(s), None, C.byref(zd),
                                          out.ctypes.data, F32, 0)
    else:
        rc = p._lib.bgs_render_ex(p._ctx, h._h, C.byref(view.to_abi()), C.byref(u), C.byref(s), None, out.ctypes.data, F32, 0)
    assert rc == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)
    if flags & abi.BGS_FLAG_ASYNC:
        assert p.sync()
    return out


def oracle_frame(cloud, h, st, view, depth=None, box=True):
    u = B.GaussianSplattingPlugin.cloud_uniform(st, None, h.aabb)
    entry = (cloud, u, (st.time_start, st.time_stop)) if st.gaussian_mode == B.GaussianMode.Gaussian4d else (cloud, u, False)
    return EO.frame([entry], view.to_abi(), [st.to_abi()], [st.num_classes], entity_flags=[1 if box else 0],
                    scene=None if depth is None else depth.cpu().numpy())


def mask(img):
    return img[..., 3] == np.float32(1.0)


def check(img, want, min_edges=1):
    """The edge mask bit for bit, the colour within PIXEL_TOL."""
    m = mask(img)
    assert int(m.sum()) >= min_edges
    bad = m != want["edge_mask"]
    assert not bad.any(), f"{int(bad.sum())} pixels' edge decisions differ, first {np.argwhere(bad)[:5].tolist()}"
    err = float(np.abs(img[..., :3] - want["image"][..., :3]).max())
    assert err <= PIXEL_TOL, err


@pytest.mark.parametrize("geom", ["obb3d", "obb2d", "aabb3d", "aabb2d"])
@pytest.mark.parametrize("with_depth", [False, True])
def test_band_edges_match_the_oracle(oracle, geom, with_depth):
    """Knife splats whose target pixels lie within a few ulps of the band edges, on both axes and thresholds: the GPU's
    edge mask is the oracle's, with and without a depth buffer; the queued frame is the synchronous one."""
    case = BX.band_case(oracle, geom)
    view, st = case.view, case.settings
    w, hh = int(view.width), int(view.height)
    p = B.GaussianSplattingPlugin(0)
    try:
        h = p.add_cloud(case.cloud)
        depth = _depth(hh, w, 3, 0.05) if with_depth else None
        img = render(p, h, st, view, BOX | PREMUL | abi.BGS_FLAG_NO_CHUNKS, depth)
        want = oracle_frame(case.cloud, h, st, view, depth)
        check(img, want, min_edges=len(case.knife_ids))
        assert np.array_equal(p.tile_ranges(), want["tile_ranges"])
        assert np.array_equal(p.tile_entries(), want["tile_entries"])
        # the knife pixels are decided on both sides of the band edge
        kp = mask(img)[case.pixels[:, 1], case.pixels[:, 0]]
        if not with_depth:
            assert kp.any() and (~kp).any()
        q = render(p, h, st, view, BOX | PREMUL | abi.BGS_FLAG_NO_CHUNKS | abi.BGS_FLAG_ASYNC, depth)
        assert q.tobytes() == img.tobytes()
        # the opaque output mode draws the same colour
        opaque = render(p, h, st, view, BOX | abi.BGS_FLAG_NO_CHUNKS, depth)
        assert opaque[..., :3].tobytes() == img[..., :3].tobytes()
    finally:
        p.destroy()


def _performer_settings(**kw):
    return S4.settings_4d(B.CloudSettings(aabb=True, global_opacity=0.9, **kw), 0.45, -0.2, 1.1)


VIEW = B.headless_view(200, 120)


@pytest.mark.parametrize("with_depth", [False, True])
def test_4d_aabb_and_4d_in_scenes(with_depth):
    """A Gaussian4d cloud with aabb (conic records) matches the oracle's edge mask, alone and inside
    bgs_render_scene_4d."""
    perf = S4.performer(6000, 9)
    st = _performer_settings()
    p = B.GaussianSplattingPlugin(0)
    try:
        h = p.add_cloud(perf)
        depth = _depth(120, 200, 5, 0.04) if with_depth else None
        img = render(p, h, st, VIEW, BOX | PREMUL | abi.BGS_FLAG_NO_CHUNKS, depth)
        want = oracle_frame(perf, h, st, VIEW, depth)
        check(img, want, min_edges=50)
        # the scene call of the one cloud: the same frame
        u = p.cloud_uniform(st, None, h.aabb)
        s = st.to_abi()
        s.gaussian_mode = int(B.GaussianMode.Gaussian3d)
        s.flags |= BOX | PREMUL | abi.BGS_FLAG_NO_CHUNKS
        out = np.empty_like(img)
        clouds = (C.c_void_p * 1)(h._h.value)
        ua = (abi.bgs_cloud_uniform * 1)(u)
        wa = (abi.bgs_time_window * 1)(abi.bgs_time_window(st.time_start, st.time_stop))
        zd = _zd(depth, 200)
        assert p._lib.bgs_render_scene_4d(p._ctx, clouds, ua, wa, 1, C.byref(VIEW.to_abi()), C.byref(s), None,
                                          None if zd is None else C.byref(zd), out.ctypes.data, F32, 0) == abi.BGS_OK
        assert out.tobytes() == img.tobytes()
    finally:
        p.destroy()


def test_invisible_splats_show_their_boxes():
    """Boxes are drawn before the opacity: opacity 0 and global_opacity 0 frames show them, as do a Velocity frame's
    zeroed splats; under DrawMode::Selected the unselected splats have no quad and no box."""
    cloud = B.random_gaussians_3d_seeded(3000, 4)
    zero = B.PlanarGaussian3d(cloud.position_visibility, cloud.spherical_harmonic, cloud.rotation,
                              np.concatenate([cloud.scale_opacity[:, :3], np.zeros((len(cloud), 1), np.float32)], 1))
    view = B.headless_view(160, 128)
    p = B.GaussianSplattingPlugin(0)
    try:
        hz, hc = p.add_cloud(zero), p.add_cloud(cloud)
        # (a fixed cutoff: the adaptive radius of an opacity-0 splat is the cutoff floor)
        for h, c, st in ((hz, zero, B.CloudSettings(global_scale=0.3, opacity_adaptive_radius=False)),
                         (hc, cloud, B.CloudSettings(global_scale=0.3, global_opacity=0.0, opacity_adaptive_radius=False)),
                         (hc, cloud, B.CloudSettings(global_scale=0.3, aabb=True, global_opacity=0.0,
                                                     opacity_adaptive_radius=False))):
            img = render(p, h, st, view, BOX | PREMUL | abi.BGS_FLAG_NO_CHUNKS)
            want = oracle_frame(c, h, st, view)
            check(img, want, min_edges=100)
            # only edges blend: every pixel is either an edge or untouched
            assert (img[~mask(img)] == 0).all()
        # Selected: half of the splats unselected (visibility 0); none selected draws no box at all
        sel = B.CloudSettings(global_scale=0.3, draw_mode=B.DrawMode.Selected)
        pv = cloud.position_visibility.copy()
        pv[::2, 3] = 0.0
        half = B.PlanarGaussian3d(pv, cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity)
        hh = p.add_cloud(half)
        img = render(p, hh, sel, view, BOX | PREMUL | abi.BGS_FLAG_NO_CHUNKS)
        check(img, oracle_frame(half, hh, sel, view), min_edges=10)
        pv[:, 3] = 0.0
        hn = p.add_cloud(B.PlanarGaussian3d(pv, cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity))
        img = render(p, hn, sel, view, BOX | PREMUL | abi.BGS_FLAG_NO_CHUNKS)
        assert not img.any()
        # Velocity: the 4D cloud's splats are drawn with zeroed colour; their boxes still show
        perf = S4.performer(4000, 9)
        hp = p.add_cloud(perf)
        vel = S4.settings_4d(B.CloudSettings(rasterize_mode=B.RasterizeMode.Velocity), 0.45, -0.2, 1.1)
        img = render(p, hp, vel, VIEW, BOX | PREMUL | abi.BGS_FLAG_NO_CHUNKS)
        check(img, oracle_frame(perf, hp, vel, VIEW), min_edges=50)
    finally:
        p.destroy()


def test_aux_frames_share_the_edge_mask():
    """bgs_render_aux: the colour, depth and normal frames carry the same edges, the colour frame's (and mask) the
    oracle's."""
    cloud = B.random_gaussians_3d_seeded(5000, 2)
    view = B.headless_view(192, 128)
    st = B.CloudSettings(global_scale=0.4)
    p = B.GaussianSplattingPlugin(0)
    try:
        h = p.add_cloud(cloud)
        u = p.cloud_uniform(st, None, h.aabb)
        s = st.to_abi()
        s.flags |= BOX | PREMUL
        frames = [np.empty((128, 192, 4), np.float32) for _ in range(3)]
        assert p._lib.bgs_render_aux(p._ctx, h._h, C.byref(view.to_abi()), C.byref(u), C.byref(s),
                                     *[f.ctypes.data for f in frames], F32, 0) == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)
        m = mask(frames[0])
        assert m.sum() > 100
        for f in frames[1:]:
            assert np.array_equal(mask(f), m)
        check(frames[0], oracle_frame(cloud, h, st, view), min_edges=100)
    finally:
        p.destroy()


def test_large_footprint_frame_renders_in_one_round(oracle):
    """A frame of big splats (what takes raster2_kernel, and chunked rounds under BGS_FLAG_CHUNKS) renders in one round
    with the overlay, matches the oracle, and its stats are the BGS_FLAG_NO_CHUNKS frame's."""
    case = BC.knife_case(oracle, "obb3d", False, heavy=True)
    view, st = case.view, dataclasses.replace(case.settings, binning_rounds=None)
    p = B.GaussianSplattingPlugin(0)
    try:
        h = p.add_cloud(case.cloud)
        render(p, h, st, view, abi.BGS_FLAG_CHUNKS)          # (the hints of a large-footprint frame)
        assert p.frame_stats().rounds > 1
        chunked = render(p, h, st, view, BOX | PREMUL | abi.BGS_FLAG_CHUNKS)
        fs = bytes(p.frame_stats())
        assert p.frame_stats().rounds == 1
        ranges, entries = p.tile_ranges(), p.tile_entries()
        one = render(p, h, st, view, BOX | PREMUL | abi.BGS_FLAG_NO_CHUNKS)
        assert bytes(p.frame_stats()) == fs
        assert one.tobytes() == chunked.tobytes()
        want = oracle_frame(case.cloud, h, st, view)
        check(one, want, min_edges=100)
        assert np.array_equal(ranges, want["tile_ranges"]) and np.array_equal(entries, want["tile_entries"])
    finally:
        p.destroy()


def test_scene_subsets_equal_the_whole():
    """A cloud split into contiguous subsets renders through bgs_render_scene byte for byte like the whole, overlay on."""
    cloud = B.random_gaussians_3d_seeded(6000, 12)
    view = B.headless_view(200, 120)
    for st in (B.CloudSettings(global_scale=0.4), B.CloudSettings(global_scale=0.4, aabb=True)):
        p = B.GaussianSplattingPlugin(0)
        try:
            h = p.add_cloud(cloud)
            whole = render(p, h, st, view, BOX | PREMUL | abi.BGS_FLAG_NO_CHUNKS)
            cuts = [0, 1000, 3500, 6000]
            parts = [B.PlanarGaussian3d(*(getattr(cloud, k)[a:b] for k in ("position_visibility", "spherical_harmonic",
                                                                             "rotation", "scale_opacity")))
                     for a, b in zip(cuts, cuts[1:])]
            hs = [p.add_cloud(c) for c in parts]
            k = len(hs)
            clouds = (C.c_void_p * k)(*[x._h.value for x in hs])
            ua = (abi.bgs_cloud_uniform * k)(*[p.cloud_uniform(st, None, h.aabb) for _ in hs])
            s = st.to_abi()
            s.flags |= BOX | PREMUL | abi.BGS_FLAG_NO_CHUNKS
            out = np.empty_like(whole)
            assert p._lib.bgs_render_scene(p._ctx, clouds, ua, k, C.byref(view.to_abi()), C.byref(s), None, None,
                                            out.ctypes.data, F32, 0) == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)
            assert mask(whole).sum() > 100
            assert out.tobytes() == whole.tobytes()
        finally:
            p.destroy()


# ---- entities

W, H = 200, 120


def _load(p, case):
    handles, unis, sts, listed, up = [], [], [], [], {}
    for cloud, layout, tr, st in E.entities(case):
        if id(cloud) not in up:
            up[id(cloud)] = p.add_cloud(cloud, f16=layout in ("f16", "cov"), precompute_covariance=layout == "cov")
        h = up[id(cloud)]
        handles.append(h)
        unis.append(p.cloud_uniform(st, tr, h.aabb))
        sts.append(st)
        listed.append(E.oracle_entry(cloud, layout, unis[-1], st))
    return handles, unis, sts, listed


def render_entities(p, handles, unis, sts, flags=0, eflags=None, depth=None, out=None, plain=False):
    k = len(handles)
    clouds = (C.c_void_p * k)(*[h._h.value for h in handles])
    ua = (abi.bgs_cloud_uniform * k)(*unis)
    ea = (abi.bgs_entity_settings * k)(*[entity_settings(st) for st in sts])
    s = sts[0].to_abi()
    s.flags |= flags
    zd = _zd(depth, W)
    tail = (C.byref(VIEW.to_abi()), C.byref(s), None, None if zd is None else C.byref(zd), out.ctypes.data, F32, 0)
    if plain:
        return p._lib.bgs_render_entities(p._ctx, clouds, ua, ea, k, *tail)
    fl = None if eflags is None else (C.c_uint32 * k)(*eflags)
    return p._lib.bgs_render_entities_ex(p._ctx, clouds, ua, ea, fl, k, *tail)


def capture(p, out):
    torch.cuda.synchronize()
    fs = p.frame_stats()
    got = {"frame": out.tobytes(), "sorted": p.sorted_entries().tobytes(), "stats": bytes(fs), "launches": p.last_launch_count}
    rec, ids = p.projected()
    got["records"], got["ids"] = rec.tobytes(), ids.tobytes()
    if fs.rounds == 1:
        got["ranges"], got["entries"] = p.tile_ranges().tobytes(), p.tile_entries().tobytes()
    return got


@pytest.mark.parametrize("case", ["kinds", "agree"])
def test_entities_ex_without_flags_is_render_entities(case):
    """bgs_render_entities_ex(..., NULL) and with all-zero flags are bgs_render_entities byte for byte: pixels, hooks,
    stats and launch count."""
    got = []
    for mode in ("plain", "null", "zeros"):
        p = B.GaussianSplattingPlugin(0)
        try:
            handles, unis, sts, _ = _load(p, case)
            out = np.empty((H, W, 4), np.float32)
            eflags = [0] * len(sts) if mode == "zeros" else None
            assert render_entities(p, handles, unis, sts, abi.BGS_FLAG_NO_CHUNKS, eflags, out=out,
                                   plain=mode == "plain") == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)
            got.append(capture(p, out))
        finally:
            p.destroy()
    for g in got[1:]:
        for key in got[0]:
            assert g[key] == got[0][key], key


FLAG_SETS = [("kinds", [1, 0, 0, 1, 0, 1]), ("kinds", [0, 1, 1, 0, 1, 0]), ("agree", [1, 0, 0, 0, 1, 0]),
             ("agree_aabb", [0, 0, 1, 0, 0, 0]), ("surfel_4d", [1, 1, 1, 1, 1, 1])]


@pytest.mark.parametrize("which", range(len(FLAG_SETS)))
@pytest.mark.parametrize("with_depth", [False, True])
def test_only_flagged_entities_draw_boxes(which, with_depth):
    """Entities with the overlay bit draw boxes, the others none: the edge mask is the entity oracle's, with and without
    a depth buffer, including entities that differ only in the bit (the mixed blend of one kind); queued is synchronous;
    the frame flag equals every bit set."""
    case, eflags = FLAG_SETS[which]
    p = B.GaussianSplattingPlugin(0)
    try:
        handles, unis, sts, listed = _load(p, case)
        depth = _depth(H, W, 7, 0.04) if with_depth else None
        img = np.empty((H, W, 4), np.float32)
        assert render_entities(p, handles, unis, sts, PREMUL | abi.BGS_FLAG_NO_CHUNKS, eflags, depth, img) == abi.BGS_OK, \
            p._lib.bgs_last_error(p._ctx)
        want = EO.frame(listed, VIEW.to_abi(), [st.to_abi() for st in sts], [st.num_classes for st in sts],
                        scene=None if depth is None else depth.cpu().numpy(), entity_flags=eflags)
        check(img, want, min_edges=20)
        assert np.array_equal(p.tile_entries(), want["tile_entries"])
        q = np.empty_like(img)
        assert render_entities(p, handles, unis, sts, PREMUL | abi.BGS_FLAG_NO_CHUNKS | abi.BGS_FLAG_ASYNC, eflags, depth,
                               q) == abi.BGS_OK
        assert p.sync()
        assert q.tobytes() == img.tobytes()
        if all(eflags):
            f = np.empty_like(img)
            assert render_entities(p, handles, unis, sts, BOX | PREMUL | abi.BGS_FLAG_NO_CHUNKS, None, depth, f) == abi.BGS_OK
            assert f.tobytes() == img.tobytes()
    finally:
        p.destroy()


def test_compare_aabb_obb_pair():
    """The reference's tools/compare_aabb_obb.rs: one cloud drawn twice side by side, one entity with aabb and one
    without, both with the overlay: the entity oracle's frame."""
    cloud = B.random_gaussians_3d_seeded(4000, 21)
    p = B.GaussianSplattingPlugin(0)
    try:
        h = p.add_cloud(cloud)
        sts = [B.CloudSettings(aabb=True, global_scale=0.5, visualize_bounding_box=True),
               B.CloudSettings(aabb=False, global_scale=0.5, visualize_bounding_box=True)]
        trs = [SC.transform((-1.2, 0.0, 0.0)), SC.transform((1.2, 0.0, 0.0))]
        view = B.headless_view(256, 160)
        img = p.render_entities([(h, st, tr) for st, tr in zip(sts, trs)], view, premultiplied=True)
        unis = [p.cloud_uniform(st, tr, h.aabb) for st, tr in zip(sts, trs)]
        want = EO.frame([(cloud, u, False) for u in unis], view.to_abi(), [st.to_abi() for st in sts], [1, 1],
                        entity_flags=[1, 1])
        check(img, want, min_edges=200)
    finally:
        p.destroy()


def test_unknown_entity_flag_is_refused():
    p = B.GaussianSplattingPlugin(0)
    try:
        handles, unis, sts, _ = _load(p, "kinds")
        for bad in (2, 0x80000000, 3):
            out = np.full((H, W, 4), 0.5, np.float32)
            flags = [0] * len(sts)
            flags[len(sts) - 1] = bad
            assert render_entities(p, handles, unis, sts, 0, flags, out=out) == abi.BGS_EINVAL
            assert (out == 0.5).all()
    finally:
        p.destroy()
