"""bgs_render_scene_4d on the H100: a Gaussian4d cloud split into contiguous subsets renders exactly like bgs_render_4d
of the whole cloud; with no 4D cloud the call is bgs_render_scene; a 4D performer inside a 3D room matches the
scene4d oracle; 3D clouds in a Velocity frame draw nothing; launch counts; a queued particle step on the 4D cloud is
seen; refusals write nothing."""
import ctypes as C

import numpy as np
import pytest
import torch

import bevy_gaussian_splatting_b200 as B
import project_cases as PC
import scene4d_cases as S4
import scene_cases as SC
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.particles import random_particle_behaviors
from scene4d_oracle import scene4d_oracle as S4O

pytestmark = pytest.mark.gpu

PIXEL_TOL = 1e-3
W, H = 200, 120
VIEW = B.headless_view(W, H)
PREV = B.perspective_view((0.2, 1.4, 5.2), (0.0, 1.5, 4.0), W, H)
FORMATS = [(abi.BGS_FORMAT_RGBA8_SRGB, np.uint8, torch.uint8), (abi.BGS_FORMAT_RGBA16F, np.float16, torch.float16),
           (abi.BGS_FORMAT_RGBA32F, np.float32, torch.float32)]
M = B.RasterizeMode


def _add(plugin, cloud, layout):
    return plugin.add_cloud(cloud, f16=layout != "f32", precompute_covariance=layout == "cov")


def _extras(mode):
    if mode not in (M.Classification, M.OpticalFlow):
        return None
    ex = abi.bgs_render_extras(num_classes=5)
    ex.previous_clip_from_world[:] = PREV.to_abi().clip_from_world[:]
    ex.delta_time = 1.0 / 60.0
    return ex


def _target(fmt, device, fill):
    _, np_t, torch_t = FORMATS[fmt]
    if device:
        return torch.full((H, W, 4), fill, dtype=torch_t, device="cuda")
    return np.full((H, W, 4), fill, np_t)


def _ptr(t):
    return t.data_ptr() if isinstance(t, torch.Tensor) else t.ctypes.data


def _code(out):
    i = 2 if isinstance(out, torch.Tensor) else 1
    return next(f[0] for f in FORMATS if out.dtype == f[i])


def _zd(depth):
    return None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * W)


def render_4d(plugin, h, u, s, ex, depth, out, device, window):
    return plugin._lib.bgs_render_4d(plugin._ctx, h._h, C.byref(VIEW.to_abi()), C.byref(u), C.byref(s),
                                     None if ex is None else C.byref(ex), None if depth is None else C.byref(_zd(depth)),
                                     _ptr(out), _code(out), int(device), C.c_float(window[0]), C.c_float(window[1]))


def render_scene_4d(plugin, handles, unis, windows, s, ex=None, depth=None, out=None, device=False, k=None):
    """windows: a list of (time_start, time_stop), or None for a NULL array."""
    k = len(handles) if k is None else k
    clouds = (C.c_void_p * max(len(handles), 1))(*[None if h is None else h._h.value for h in handles])
    ua = (abi.bgs_cloud_uniform * max(len(unis), 1))(*unis)
    wa = None if windows is None else (abi.bgs_time_window * max(len(windows), 1))(*[abi.bgs_time_window(*w) for w in windows])
    return plugin._lib.bgs_render_scene_4d(plugin._ctx, clouds, ua, wa, k, C.byref(VIEW.to_abi()), C.byref(s),
                                           None if ex is None else C.byref(ex), None if depth is None else C.byref(_zd(depth)),
                                           None if out is None else _ptr(out), _code(out) if out is not None else 0, int(device))


def render_scene(plugin, handles, unis, s, ex=None, depth=None, out=None, device=False):
    clouds = (C.c_void_p * len(handles))(*[h._h.value for h in handles])
    ua = (abi.bgs_cloud_uniform * len(unis))(*unis)
    return plugin._lib.bgs_render_scene(plugin._ctx, clouds, ua, len(handles), C.byref(VIEW.to_abi()), C.byref(s),
                                        None if ex is None else C.byref(ex), None if depth is None else C.byref(_zd(depth)),
                                        _ptr(out), _code(out), int(device))


def capture(plugin, out, depth_tested):
    """Everything a frame reports: pixels, sorted entries, tile ranges and slices, records, stats, launches."""
    torch.cuda.synchronize()
    fs = plugin.frame_stats()
    got = {"frame": (out.cpu().numpy() if isinstance(out, torch.Tensor) else out).tobytes(),
           "sorted": plugin.sorted_entries().tobytes(), "stats": bytes(fs), "launches": plugin.last_launch_count}
    rec, ids = plugin.projected()
    got["records"], got["ids"] = rec.tobytes(), ids.tobytes()
    if fs.rounds == 1:
        got["ranges"], got["entries"] = plugin.tile_ranges().tobytes(), plugin.tile_entries().tobytes()
    if depth_tested:
        got["splat_depths"] = plugin.splat_depths().tobytes()
    return got


def _cases():
    modes = [M.Color, M.Depth, M.Position, M.Classification, M.OpticalFlow, M.Velocity]
    out = []
    for i in range(18):
        mode = modes[i % len(modes)]
        flags = [abi.BGS_FLAG_NO_CHUNKS, abi.BGS_FLAG_CHUNKS][(i // 3) % 2]
        blend = i % 5 == 1
        if blend:
            flags |= abi.BGS_FLAG_BLEND_OVER_TARGET
        elif i % 5 == 2:
            flags |= abi.BGS_FLAG_PREMULTIPLIED_OUT
        out.append(dict(id=f"{i}-{mode.name}", mode=mode, aabb=i % 4 >= 2, draw=B.DrawMode(i % 3), fmt=(i // 2) % 3,
                        device=blend or i % 2 == 1, depth=i % 3 == 0, flags=flags, asynchronous=i % 6 == 5, seed=i,
                        time=(0.15, 0.5, 0.85)[i % 3]))
    return out


CASES = _cases()


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_split_4d_cloud_renders_like_render_4d(case):
    cloud = S4.performer(4000, case["seed"])
    st = S4.settings_4d(B.CloudSettings(rasterize_mode=case["mode"], aabb=case["aabb"], draw_mode=case["draw"], num_classes=5),
                        case["time"], -0.1, 1.2)
    s = st.to_abi()
    s.flags |= case["flags"]
    ex = _extras(case["mode"])
    window = (st.time_start, st.time_stop)
    tr = SC.transform((0.2, -0.1, 0.3), 1.05, 0.3)
    depth = None
    if case["depth"]:
        g = torch.Generator(device="cuda").manual_seed(case["seed"])
        depth = torch.rand((H, W), generator=g, device="cuda") * 0.04
    p0 = B.GaussianSplattingPlugin(0)
    try:
        h = p0.add_cloud(cloud)
        u = p0.cloud_uniform(st, tr, h.aabb)
        other = _add(p0, SC.cloud_in_box(500, 99), "f32")
        ou = p0.cloud_uniform(B.CloudSettings(), None, other.aabb)
        s_async = abi.bgs_settings.from_buffer_copy(bytes(s))
        s_async.flags |= abi.BGS_FLAG_ASYNC
        s_other = B.CloudSettings().to_abi()
        s_other.flags |= abi.BGS_FLAG_ASYNC

        def frame(render):
            out = _target(case["fmt"], case["device"], 0.25 if FORMATS[case["fmt"]][0] else 64)
            if case["asynchronous"]:
                # queued between single-cloud frames of another cloud
                o2 = _target(case["fmt"], True, 0)
                assert p0._lib.bgs_render(p0._ctx, other._h, C.byref(VIEW.to_abi()), C.byref(ou), C.byref(s_other), _ptr(o2),
                                          FORMATS[case["fmt"]][0], 1) == abi.BGS_OK
                assert render(s_async, out) == abi.BGS_OK
                assert p0._lib.bgs_render(p0._ctx, other._h, C.byref(VIEW.to_abi()), C.byref(ou), C.byref(s_other), _ptr(o2),
                                          FORMATS[case["fmt"]][0], 1) == abi.BGS_OK
                assert p0.sync()
                assert render(s_async, out) == abi.BGS_OK   # (the hooks report the last frame: this one)
                assert p0.sync()
            else:
                assert render(s, out) == abi.BGS_OK, p0._lib.bgs_last_error(p0._ctx)
            return capture(p0, out, depth is not None)

        want = frame(lambda s_, out: render_4d(p0, h, u, s_, ex, depth, out, case["device"], window))
        rec = np.frombuffer(want["records"], np.float32).reshape(-1, 12)
        assert 0 < S4.drawn(rec).sum() < len(rec)   # part of the cloud is masked by time
        for k in (1, 2, 3, 7):
            parts = [p0.subset(h, ix) for ix in SC.pieces(len(cloud), k, case["seed"])]
            try:
                got = frame(lambda s_, out: render_scene_4d(p0, parts, [u] * k, [window] * k, s_, ex, depth, out, case["device"]))
            finally:
                for q in parts:
                    q.destroy()
            for key in want:
                assert got[key] == want[key], f"k={k}: {key} differs from bgs_render_4d's"
    finally:
        p0.destroy()


@pytest.mark.parametrize("i", [0, 5, 7, 9, 13])
def test_no_4d_cloud_is_render_scene(i):
    """A 3D-only list: bgs_render_scene exactly, with windows NULL and with garbage windows (never read)."""
    layouts = [("f32", 3), ("f16", 1), ("cov", 0), ("f32", 2), ("f16", 3)]
    modes = [M.Color, M.Depth, M.Normal, M.Position, M.OpticalFlow]
    layout, deg = layouts[i % 5]
    mode = M.Color if layout == "cov" else modes[(i // 2) % 5]
    st = B.CloudSettings(rasterize_mode=mode, aabb=i % 2 == 1, gaussian_mode=B.GaussianMode.Gaussian2d if i == 13 else B.GaussianMode.Gaussian3d)
    s = st.to_abi()
    s.flags |= abi.BGS_FLAG_NO_CHUNKS
    ex = _extras(mode)
    depth = torch.rand((H, W), generator=torch.Generator(device="cuda").manual_seed(i), device="cuda") * 0.04 if i % 2 == 0 else None
    p = B.GaussianSplattingPlugin(0)
    try:
        cloud = SC.cloud_in_box(4000, i, sh_degree=deg)
        h = _add(p, cloud, layout)
        u = p.cloud_uniform(st, SC.transform((0.1, 0.0, 0.2)), h.aabb)
        parts = [p.subset(h, ix) for ix in SC.pieces(len(cloud), 3, i)]
        out = np.zeros((H, W, 4), np.float32)
        assert render_scene(p, parts, [u] * 3, s, ex, depth, out) == abi.BGS_OK
        want = capture(p, out, depth is not None)
        for windows in (None, [(float("nan"), float("nan"))] * 3, [(1.0, 1.0)] * 3):
            out = np.zeros((H, W, 4), np.float32)
            assert render_scene_4d(p, parts, [u] * 3, windows, s, ex, depth, out) == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)
            got = capture(p, out, depth is not None)
            for key in want:
                assert got[key] == want[key], key
    finally:
        p.destroy()


def _mixed(p, mode, aabb, t0=0.35, t1=0.8):
    """The room (S4.room) plus the performer, listed twice: at t0 in place, and at t1 with another transform."""
    handles, unis, windows, listed = [], [], [], []
    for cloud, layout, _, tr, kw in S4.room():
        h = _add(p, cloud, layout)
        st = B.CloudSettings(rasterize_mode=mode, aabb=aabb, **kw)
        handles.append(h)
        unis.append(p.cloud_uniform(st, tr, h.aabb))
        windows.append((float("nan"), 0.0))   # (never read for a 3D cloud)
        listed.append((SC.oracle_cloud(cloud, layout), unis[-1], layout == "cov"))
    perf = S4.performer(5000, 9)
    h4 = p.add_cloud(perf)
    for t, tr in ((t0, None), (t1, SC.transform((0.4, 0.1, -0.3), 1.1, 0.9))):
        st = S4.settings_4d(B.CloudSettings(rasterize_mode=mode, aabb=aabb, global_opacity=0.9), t, -0.2, 1.1)
        handles.append(h4)
        unis.append(p.cloud_uniform(st, tr, h4.aabb))
        windows.append((st.time_start, st.time_stop))
        listed.append((perf, unis[-1], (st.time_start, st.time_stop)))
    return handles, unis, windows, listed, perf


@pytest.mark.parametrize("mode", [M.Color, M.Depth, M.Position, M.Velocity])
@pytest.mark.parametrize("aabb", [False, True])
def test_mixed_scene_matches_the_scene4d_oracle(mode, aabb):
    p = B.GaussianSplattingPlugin(0)
    try:
        handles, unis, windows, listed, perf = _mixed(p, mode, aabb)
        s = B.CloudSettings(rasterize_mode=mode, aabb=aabb).to_abi()
        s.flags |= abi.BGS_FLAG_NO_CHUNKS
        img = np.empty((H, W, 4), np.float32)
        assert render_scene_4d(p, handles, unis, windows, s, out=img) == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)
        want = S4O.frame(listed, VIEW.to_abi(), s)
        assert np.array_equal(p.sorted_entries(), want["sorted"])
        fs = p.frame_stats()
        assert fs.n == sum(len(c) for c, _, _ in listed) and fs.n_visible == want["n_vis"]
        assert np.array_equal(p.tile_ranges(), want["tile_ranges"])
        assert np.array_equal(p.tile_entries(), want["tile_entries"])
        rec, ids = p.projected()
        assert np.array_equal(ids, want["rank_to_id"])
        n3 = sum(len(c) for c, _, _ in listed[:-2])
        four = ids >= n3
        orec = want["records"]
        geo = [0, 1, 2, 3, 4, 5, 6, 7, 11]
        assert PC.bits_agree(rec[four][:, geo], orec[four][:, geo]).all()
        if mode == M.Color:
            d = four & S4.drawn(rec)
            local = (ids[d] - n3) % len(perf)
            err = np.abs(rec[d, 8:11].astype(np.float64) - orec[d, 8:11])
            assert (err <= S4.sh_bound(perf, local)).all(), err.max()
        else:
            assert PC.bits_agree(rec[four][:, 8:11], orec[four][:, 8:11]).all()
        if mode == M.Velocity:   # the room's gaussians: counted and sorted, but undrawn and in no tile
            three = ~four
            assert three.any() and not S4.drawn(rec[three]).any()
            assert (rec[three][:, 8:11] == 0).all()
            assert not np.isin(p.tile_entries(), np.flatnonzero(three)).any()
        assert float(np.abs(img - want["image"]).max()) <= PIXEL_TOL
    finally:
        p.destroy()


def test_depth_tested_mixed_scene_matches_the_scene4d_oracle():
    """Splat depths: the room's from the base positions, the performer's from the moved ones."""
    p = B.GaussianSplattingPlugin(0)
    try:
        handles, unis, windows, listed, _ = _mixed(p, M.Color, False)
        s = B.CloudSettings().to_abi()
        s.flags |= abi.BGS_FLAG_NO_CHUNKS
        depth = torch.rand((H, W), generator=torch.Generator(device="cuda").manual_seed(3), device="cuda") * 0.04
        img = np.empty((H, W, 4), np.float32)
        assert render_scene_4d(p, handles, unis, windows, s, depth=depth, out=img) == abi.BGS_OK
        want = S4O.frame(listed, VIEW.to_abi(), s, scene=depth.cpu().numpy())
        assert PC.bits_agree(p.splat_depths(), want["depths"]).all()
        assert float(np.abs(img - want["image"]).max()) <= PIXEL_TOL
    finally:
        p.destroy()


def test_launch_counts():
    p = B.GaussianSplattingPlugin(0)
    try:
        out = np.empty((H, W, 4), np.float32)
        depth = torch.zeros((H, W), device="cuda")
        room = [(_add(p, c, layout), tr, kw) for c, layout, _, tr, kw in S4.room()]
        st = B.CloudSettings()
        rh = [h for h, _, _ in room]
        ru = [p.cloud_uniform(B.CloudSettings(**kw), tr, h.aabb) for h, tr, kw in room]
        perf = S4.performer(5000, 9)
        h4 = p.add_cloud(perf)
        st4 = S4.settings_4d(st, 0.4)
        u4 = p.cloud_uniform(st4, None, h4.aabb)
        w4 = (st4.time_start, st4.time_stop)
        for zd in (None, depth):
            s = st.to_abi()
            s.flags |= abi.BGS_FLAG_NO_CHUNKS
            assert render_scene(p, rh, ru, s, depth=zd, out=out) == abi.BGS_OK
            room_only = p.last_launch_count
            assert render_scene_4d(p, rh + [h4, h4], ru + [u4, u4], [w4] * 6, s, depth=zd, out=out) == abi.BGS_OK
            assert p.last_launch_count == room_only + 1
            s4 = st4.to_abi()
            s4.flags |= abi.BGS_FLAG_NO_CHUNKS
            assert render_4d(p, h4, u4, s4, None, zd, out, False, w4) == abi.BGS_OK
            one = p.last_launch_count
            parts = [p.subset(h4, ix) for ix in SC.pieces(len(perf), 5)]
            assert render_scene_4d(p, parts + [h4], [u4] * 6, [w4] * 6, s4, depth=zd, out=out) == abi.BGS_OK
            assert p.last_launch_count == one
    finally:
        p.destroy()


def test_scene_reads_the_4d_cloud_after_a_particle_step_on_another_context():
    p, q = B.GaussianSplattingPlugin(0), B.GaussianSplattingPlugin(0)
    try:
        room_cloud = SC.cloud_in_box(3000, 11, centre=S4.ROOM_CENTRE, half=1.2)
        perf = S4.performer(3000, 12)
        a, h4 = _add(p, room_cloud, "f32"), p.add_cloud(perf)
        st = B.CloudSettings()
        st4 = S4.settings_4d(st, 0.5)
        s = st.to_abi()
        s.flags |= abi.BGS_FLAG_NO_CHUNKS
        u, u4, w4 = p.cloud_uniform(st, None, a.aabb), p.cloud_uniform(st4, None, h4.aabb), (st4.time_start, st4.time_stop)
        beh = q.add_particles(random_particle_behaviors(3000, 3))
        q.step_particles(h4, beh, 0.5)   # queued on q; the frame on p must see it
        got = np.empty((H, W, 4), np.float32)
        assert render_scene_4d(p, [a, h4], [u, u4], [(0.0, 0.0), w4], s, out=got) == abi.BGS_OK
        q.sync()
        p.sync()
        moved = p.positions(h4)
        assert not np.array_equal(moved, perf.position_visibility)
        h_now = p.add_cloud(B.PlanarGaussian4d(moved, *perf.planes()[1:]))
        want = np.empty((H, W, 4), np.float32)
        assert render_scene_4d(p, [a, h_now], [u, u4], [(0.0, 0.0), w4], s, out=want) == abi.BGS_OK
        assert got.tobytes() == want.tobytes()
    finally:
        q.destroy()
        p.destroy()


def test_refusals_write_nothing():
    p = B.GaussianSplattingPlugin(0)
    try:
        st = B.CloudSettings()
        h = _add(p, SC.cloud_in_box(2000, 21), "f32")
        c4 = p.add_cloud(S4.performer(1000, 22))
        st4 = S4.settings_4d(st, 0.3)
        u, u4 = p.cloud_uniform(st, None, h.aabb), p.cloud_uniform(st4, None, c4.aabb)
        ok_w = (0.0, 1.0)
        out = torch.full((H, W, 4), 0.375, device="cuda")
        before = out.clone()

        def refused(handles, unis, windows, s_, k=None, status=abi.BGS_EINVAL):
            assert render_scene_4d(p, handles, unis, windows, s_, out=out, device=True, k=k) == status
            torch.cuda.synchronize()
            assert torch.equal(out, before)

        s = st.to_abi()
        assert render_scene_4d(p, [h, c4], [u, u4], [ok_w] * 2, s, out=out, device=True) == abi.BGS_OK   # (accepted as given)
        torch.cuda.synchronize()
        out.copy_(before)
        # bgs_render_scene's refusals
        refused([h, c4], [u, u4], [ok_w] * 2, s, k=0)
        refused([c4] * 65, [u4] * 65, [ok_w] * 65, s)
        refused([h, None], [u, u], [ok_w] * 2, s)
        s_all = st.to_abi()
        s_all.flags |= abi.BGS_FLAG_SORT_ALL
        refused([h, c4], [u, u4], [ok_w] * 2, s_all)
        # bgs_render_4d's, for the 4D cloud with its uniform and window
        for w in ((float("nan"), 1.0), (0.0, float("inf")), (0.5, 0.5), (-3e38, 3e38)):
            refused([h, c4], [u, u4], [ok_w, w], s)
        u_nan = p.cloud_uniform(S4.settings_4d(st, float("nan")), None, c4.aabb)
        refused([h, c4], [u, u_nan], [ok_w] * 2, s)
        refused([h, c4], [u, u4], [ok_w] * 2, B.CloudSettings(rasterize_mode=M.Normal).to_abi())
        # windows NULL; Gaussian4d mode with a 3D cloud; 2D with AABB and a 4D cloud
        refused([h, c4], [u, u4], None, s)
        refused([h, c4], [u, u4], [ok_w] * 2, S4.settings_4d(st, 0.3).to_abi())
        refused([h, c4], [u, u4], [ok_w] * 2, B.CloudSettings(gaussian_mode=B.GaussianMode.Gaussian2d, aabb=True).to_abi())
        # Velocity without a 4D cloud is bgs_render_scene's refusal
        refused([h], [u], None, B.CloudSettings(rasterize_mode=M.Velocity).to_abi())
        # NULL arrays, view or settings: not ready
        assert p._lib.bgs_render_scene_4d(p._ctx, None, None, None, 1, C.byref(VIEW.to_abi()), C.byref(s), None, None,
                                          out.data_ptr(), abi.BGS_FORMAT_RGBA32F, 1) == abi.BGS_NOT_READY
        torch.cuda.synchronize()
        assert torch.equal(out, before)
    finally:
        p.destroy()


def test_plugin_render_scene_takes_4d_entities():
    p = B.GaussianSplattingPlugin(0)
    try:
        room_cloud = SC.cloud_in_box(3000, 31, centre=S4.ROOM_CENTRE, half=1.2)
        perf = S4.performer(3000, 32)
        a, h4 = _add(p, room_cloud, "f16"), p.add_cloud(perf)
        st, st4 = B.CloudSettings(binning_rounds=False), S4.settings_4d(B.CloudSettings(binning_rounds=False), 0.6, 0.0, 2.0)
        got = p.render_scene([(a, st, None), (h4, st4, None), (h4, S4.settings_4d(st4, 1.4, 0.0, 2.0), SC.transform((0.3, 0.0, 0.0)))], VIEW)
        s = st.to_abi()
        u, u4 = p.cloud_uniform(st, None, a.aabb), p.cloud_uniform(st4, None, h4.aabb)
        u4b = p.cloud_uniform(S4.settings_4d(st4, 1.4, 0.0, 2.0), SC.transform((0.3, 0.0, 0.0)), h4.aabb)
        want = np.empty((H, W, 4), np.float32)
        assert render_scene_4d(p, [a, h4, h4], [u, u4, u4b], [(0.0, 0.0), (0.0, 2.0), (0.0, 2.0)], s, out=want) == abi.BGS_OK
        assert got.tobytes() == want.tobytes()
        with pytest.raises(ValueError):
            p.render_scene([(a, st, None), (h4, st, None)], VIEW)   # a 4D entity must be Gaussian4d
    finally:
        p.destroy()
