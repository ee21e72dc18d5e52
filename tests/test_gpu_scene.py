"""bgs_render_scene on the H100: a cloud split into contiguous subsets renders bit-identically to the whole cloud in
every layout, degree, geometry, mode, draw mode, format, target and flag; mixed scenes match the scene oracle; a
homogeneous scene costs the launches of one cloud; member clouds are read after the writes queued on them; refusals
write nothing; and a scene frame that outgrows the pair buffer re-renders like a single frame."""
import ctypes as C

import numpy as np
import pytest
import torch

import bevy_gaussian_splatting_b200 as B
import scene_cases as SC
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.particles import random_particle_behaviors
from scene_oracle import scene_oracle as SO

pytestmark = pytest.mark.gpu

PIXEL_TOL = 1e-3   # test_gpu_parity's per-pixel bound
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
    code, np_t, torch_t = FORMATS[fmt]
    if device:
        return torch.full((H, W, 4), fill, dtype=torch_t, device="cuda")
    return np.full((H, W, 4), fill, np_t)


def _ptr(t):
    return t.data_ptr() if isinstance(t, torch.Tensor) else t.ctypes.data


def _zd(depth):
    return None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * W)


def render_whole(plugin, h, u, s, ex, depth, out, device):
    return plugin._lib.bgs_render_depth_test(plugin._ctx, h._h, C.byref(VIEW.to_abi()), C.byref(u), C.byref(s),
                                             None if ex is None else C.byref(ex),
                                             None if depth is None else C.byref(_zd(depth)), _ptr(out), FORMATS_CODE(out), int(device))


def FORMATS_CODE(out):
    i = 2 if isinstance(out, torch.Tensor) else 1
    return next(f[0] for f in FORMATS if out.dtype == f[i])


def render_scene(plugin, handles, unis, s, ex=None, depth=None, out=None, device=False, k=None):
    k = len(handles) if k is None else k
    clouds = (C.c_void_p * max(len(handles), 1))(*[None if h is None else h._h.value for h in handles])
    ua = (abi.bgs_cloud_uniform * max(len(unis), 1))(*unis)
    return plugin._lib.bgs_render_scene(plugin._ctx, clouds, ua, k, C.byref(VIEW.to_abi()), C.byref(s),
                                        None if ex is None else C.byref(ex), None if depth is None else C.byref(_zd(depth)),
                                        None if out is None else _ptr(out), FORMATS_CODE(out) if out is not None else 0, int(device))


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
    layouts = [("f32", 3), ("f16", 3), ("cov", 3), ("f32", 0), ("f16", 1), ("f32", 2), ("f16", 0), ("cov", 1), ("f32", 1),
               ("f16", 2)]
    modes = [M.Color, M.Depth, M.Normal, M.Position, M.Classification, M.OpticalFlow]
    out = []
    for i in range(30):
        layout, deg = layouts[i % len(layouts)]
        mode = modes[i % len(modes)]
        gm = B.GaussianMode.Gaussian2d if (i % 4 == 3 and layout != "cov") else B.GaussianMode.Gaussian3d
        if layout == "cov" and mode == M.Normal:
            mode = M.Color
        flags = [abi.BGS_FLAG_NO_CHUNKS, abi.BGS_FLAG_CHUNKS][(i // 3) % 2]
        blend = i % 5 == 1
        if blend:
            flags |= abi.BGS_FLAG_BLEND_OVER_TARGET
        elif i % 5 == 2:
            flags |= abi.BGS_FLAG_PREMULTIPLIED_OUT
        out.append(dict(id=f"{i}-{layout}{deg}-{mode.name}-{gm.name}", layout=layout, deg=deg, mode=mode, gm=gm, aabb=i % 3 == 1,
                        draw=B.DrawMode(i % 3), fmt=(i // 2) % 3, device=blend or i % 2 == 1, depth=i % 4 == 0, flags=flags,
                        asynchronous=i % 6 == 5, seed=i))
    return out


CASES = _cases()


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_split_cloud_renders_bit_identically(case):
    cloud = SC.cloud_in_box(4000, case["seed"], sh_degree=case["deg"])
    st = B.CloudSettings(rasterize_mode=case["mode"], gaussian_mode=case["gm"], aabb=case["aabb"], draw_mode=case["draw"],
                         num_classes=5)
    s = st.to_abi()
    s.flags |= case["flags"]
    ex = _extras(case["mode"])
    tr = SC.transform((0.2, -0.1, 0.3), 1.05, 0.3)
    depth = None
    if case["depth"]:
        g = torch.Generator(device="cuda").manual_seed(case["seed"])
        depth = torch.rand((H, W), generator=g, device="cuda") * 0.04
    p0 = B.GaussianSplattingPlugin(0)
    try:
        h = _add(p0, cloud, case["layout"])
        u = p0.cloud_uniform(st, tr, h.aabb)
        other = _add(p0, SC.cloud_in_box(500, 99), "f32")
        ou = p0.cloud_uniform(B.CloudSettings(), None, other.aabb)
        s_async = abi.bgs_settings.from_buffer_copy(bytes(s))
        s_async.flags |= abi.BGS_FLAG_ASYNC

        def frame(render):
            out = _target(case["fmt"], case["device"], 0.25 if FORMATS[case["fmt"]][0] else 64)
            if case["asynchronous"]:
                # queued between single-cloud frames of another cloud
                o2 = _target(case["fmt"], True, 0)
                assert p0._lib.bgs_render_ex(p0._ctx, other._h, C.byref(VIEW.to_abi()), C.byref(ou), C.byref(s_async),
                                             None if ex is None else C.byref(ex), _ptr(o2), FORMATS[case["fmt"]][0], 1) == abi.BGS_OK
                assert render(s_async, out) == abi.BGS_OK
                assert p0.sync()
            else:
                assert render(s, out) == abi.BGS_OK, p0._lib.bgs_last_error(p0._ctx)
            return capture(p0, out, depth is not None)

        want = frame(lambda s_, out: render_whole(p0, h, u, s_, ex, depth, out, case["device"]))
        for k in (1, 2, 3, 7):
            parts = [p0.subset(h, ix) for ix in SC.pieces(len(cloud), k, case["seed"])]
            try:
                got = frame(lambda s_, out: render_scene(p0, parts, [u] * k, s_, ex, depth, out, case["device"]))
            finally:
                for q in parts:
                    q.destroy()
            for key in want:
                assert got[key] == want[key], f"k={k}: {key} differs from the whole cloud's"
    finally:
        p0.destroy()


@pytest.mark.parametrize("mode", [M.Color, M.Depth, M.Position])
@pytest.mark.parametrize("aabb", [False, True])
def test_mixed_scene_matches_the_scene_oracle(mode, aabb):
    """Different transforms, global_scale, global_opacity and color_space; f32, f16 and covariance clouds of several SH
    degrees, interpenetrating; one cloud listed twice with two transforms."""
    p = B.GaussianSplattingPlugin(0)
    try:
        spec = [("f32", 3, SC.transform(), dict()),
                ("f16", 1, SC.transform((0.3, 0.1, 0.2), 1.2, 0.7), dict(global_scale=1.3, global_opacity=0.8)),
                ("cov", 3, SC.transform((-0.4, 0.0, -0.2)), dict(color_space=B.GaussianColorSpace.LinRec709Display)),
                ("f32", 0, SC.transform((0.1, -0.3, 0.4), 0.8, -0.5), dict(global_opacity=0.6))]
        if mode == M.Normal:
            spec = [x for x in spec if x[0] != "cov"]
        handles, unis, listed = [], [], []
        for j, (layout, deg, tr, kw) in enumerate(spec):
            cloud = SC.cloud_in_box(3000, 40 + j, centre=(0.0, 1.5, -1.0), half=1.2, scale=0.08, sh_degree=deg)
            h = _add(p, cloud, layout)
            st = B.CloudSettings(rasterize_mode=mode, aabb=aabb, **kw)
            handles.append(h)
            unis.append(p.cloud_uniform(st, tr, h.aabb))
            listed.append((SC.oracle_cloud(cloud, layout), unis[-1], layout == "cov"))
        # the first cloud again, as an instance with its own transform
        st0 = B.CloudSettings(rasterize_mode=mode, aabb=aabb)
        handles.append(handles[0])
        unis.append(p.cloud_uniform(st0, SC.transform((0.5, 0.2, -0.6), 1.0, 1.2), handles[0].aabb))
        listed.append((listed[0][0], unis[-1], False))
        s = st0.to_abi()
        s.flags |= abi.BGS_FLAG_NO_CHUNKS
        img = np.empty((H, W, 4), np.float32)
        assert render_scene(p, handles, unis, s, out=img) == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)
        want = SO.render_tiles(listed, VIEW.to_abi(), s)
        assert np.array_equal(p.sorted_entries(), SO.sorted_entries(listed, VIEW.to_abi()))
        fs = p.frame_stats()
        assert fs.n == sum(len(c) for c, _, _ in listed) and fs.n_visible == want["n_vis"]
        assert np.array_equal(p.tile_ranges(), want["tile_ranges"])
        assert np.array_equal(p.tile_entries(), want["tile_entries"])
        assert np.array_equal(p.projected()[1], want["rank_to_id"])
        assert float(np.abs(img - want["image"]).max()) <= PIXEL_TOL
        for h in {id(h): h for h in handles}.values():
            h.destroy()
    finally:
        p.destroy()


def test_homogeneous_scene_costs_the_launches_of_one_cloud():
    p = B.GaussianSplattingPlugin(0)
    try:
        cloud = SC.cloud_in_box(20000, 7)
        st = B.CloudSettings()
        s = st.to_abi()
        s.flags |= abi.BGS_FLAG_NO_CHUNKS
        out = np.empty((H, W, 4), np.float32)
        h = _add(p, cloud, "f16")
        u = p.cloud_uniform(st, None, h.aabb)
        assert render_scene(p, [h], [u], s, out=out) == abi.BGS_OK
        one = p.last_launch_count
        parts = [p.subset(h, ix) for ix in SC.pieces(len(cloud), 64)]
        assert render_scene(p, parts, [u] * 64, s, out=out) == abi.BGS_OK
        assert p.last_launch_count == one
        f32 = _add(p, cloud, "f32")
        assert render_scene(p, parts[:32] + [f32], [u] * 33, s, out=out) == abi.BGS_OK
        assert p.last_launch_count == one + 1
        cov = _add(p, cloud, "cov")   # (f16 and covariance clouds share one projection kernel)
        assert render_scene(p, [h, cov], [u] * 2, s, out=out) == abi.BGS_OK
        assert p.last_launch_count == one
    finally:
        p.destroy()


@pytest.mark.parametrize("same_context", [True, False])
def test_scene_reads_member_clouds_after_queued_writes(same_context):
    p = B.GaussianSplattingPlugin(0)
    q = p if same_context else B.GaussianSplattingPlugin(0)
    try:
        st = B.CloudSettings()
        s = st.to_abi()
        s.flags |= abi.BGS_FLAG_NO_CHUNKS
        a_cloud, b_cloud = SC.cloud_in_box(3000, 11), SC.cloud_in_box(3000, 12)
        a, b, b2 = _add(p, a_cloud, "f32"), _add(p, b_cloud, "f32"), _add(p, SC.cloud_in_box(3000, 13), "f32")
        morph = p.subset(b, np.arange(b.n))
        u = p.cloud_uniform(st, None, a.aabb)
        beh = p.add_particles(random_particle_behaviors(3000, 3))
        # queued on q: a particle step of `a` and an interpolation into `morph`; the scene frame on p must see both
        q.step_particles(a, beh, 0.5)
        q.interpolate(morph, b, b2, B.CloudSettings(time=0.3, time_start=0.0, time_stop=1.0))
        got = np.empty((H, W, 4), np.float32)
        assert render_scene(p, [a, morph], [u, u], s, out=got) == abi.BGS_OK
        q.sync()
        p.sync()
        # the same frame from the completed clouds
        a_now = _add(p, B.PlanarGaussian3d(p.positions(a), a_cloud.spherical_harmonic, a_cloud.rotation, a_cloud.scale_opacity), "f32")
        m_now = _add(p, p.download(morph), "f32")
        want = np.empty((H, W, 4), np.float32)
        assert render_scene(p, [a_now, m_now], [u, u], s, out=want) == abi.BGS_OK
        assert got.tobytes() == want.tobytes()
        assert not np.array_equal(p.positions(a), a_cloud.position_visibility)
    finally:
        if q is not p:
            q.destroy()
        p.destroy()


def test_refusals_write_nothing():
    p = B.GaussianSplattingPlugin(0)
    try:
        st = B.CloudSettings()
        s = st.to_abi()
        h = _add(p, SC.cloud_in_box(2000, 21), "f32")
        cov = _add(p, SC.cloud_in_box(2000, 22), "cov")
        c4 = p.add_cloud(B.random_gaussians_4d_seeded(100, 0))
        u = p.cloud_uniform(st, None, h.aabb)
        out = torch.full((H, W, 4), 0.375, device="cuda")
        before = out.clone()

        def refused(handles, unis, s_, k=None, status=abi.BGS_EINVAL):
            assert render_scene(p, handles, unis, s_, out=out, device=True, k=k) == status
            torch.cuda.synchronize()
            assert torch.equal(out, before)

        refused([h], [u], s, k=0)
        refused([h] * 65, [u] * 65, s)
        refused([h, None], [u, u], s)
        refused([h, c4], [u, u], s)
        s_all = st.to_abi()
        s_all.flags |= abi.BGS_FLAG_SORT_ALL
        refused([h], [u], s_all)
        s_n = B.CloudSettings(rasterize_mode=M.Normal).to_abi()
        refused([h, cov], [u, u], s_n)
        s_2d = B.CloudSettings(gaussian_mode=B.GaussianMode.Gaussian2d).to_abi()
        refused([cov], [u], s_2d)
        # N >= 2^30: one 2^24-gaussian cloud listed 64 times
        nb = 1 << 24
        planes = [np.zeros((nb, 4), np.float32) for _ in range(4)]
        big = p.add_cloud(B.PlanarGaussian3d(*planes))
        refused([big] * 64, [u] * 64, s)
        big.destroy()
        # NULL arrays, view or settings: not ready, as bgs_render
        assert p._lib.bgs_render_scene(p._ctx, None, None, 1, C.byref(VIEW.to_abi()), C.byref(s), None, None,
                                       out.data_ptr(), abi.BGS_FORMAT_RGBA32F, 1) == abi.BGS_NOT_READY
    finally:
        p.destroy()


def test_scene_frame_that_outgrows_the_pair_buffer_re_renders_like_one_cloud():
    cloud = SC.cloud_in_box(30000, 31, centre=(0.0, 1.5, 2.0), half=2.0, scale=1.5)
    st = B.CloudSettings()
    s = st.to_abi()
    s.flags |= abi.BGS_FLAG_NO_CHUNKS
    view = B.headless_view(1280, 720)
    results = []
    for split in (False, True):
        p = B.GaussianSplattingPlugin(0)   # fresh: the first guess of the pair buffer is too small for this frame
        try:
            h = _add(p, cloud, "f16")
            u = p.cloud_uniform(st, None, h.aabb)
            hs = [p.subset(h, ix) for ix in SC.pieces(len(cloud), 5)] if split else [h]
            out = np.empty((720, 1280, 4), np.float32)
            clouds = (C.c_void_p * len(hs))(*[x._h.value for x in hs])
            ua = (abi.bgs_cloud_uniform * len(hs))(*([u] * len(hs)))
            assert p._lib.bgs_render_scene(p._ctx, clouds, ua, len(hs), C.byref(view.to_abi()), C.byref(s), None, None,
                                           out.ctypes.data, abi.BGS_FORMAT_RGBA32F, 0) == abi.BGS_OK
            fs = p.frame_stats()
            assert fs.n_pairs > (1 << 20)
            results.append((out.tobytes(), bytes(fs), p.tile_ranges().tobytes()))
        finally:
            p.destroy()
    assert results[0] == results[1]
