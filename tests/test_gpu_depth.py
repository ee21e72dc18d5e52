"""bgs_render_depth_test on the GPU (the rule: include/bgs.h; the oracle: depth_oracle/).

1. bgs_debug_splat_depths is bit-exact against the oracle's d: compact and SORT_ALL frames, 32-, 24- and 16-bit keys,
   the three cloud layouts, 2DGS and 3DGS.
2. A zero depth buffer gives the bytes of bgs_render_ex on every blend kernel (MODE 0..2's raster_kernel, raster2_kernel<false>,
   chunked raster2_kernel<true>), in each format and output mode, synchronous and queued, with the same sorted entries,
   tile ranges, tile entries and frame stats.
3. Saturated frames with knife buffers at, one ulp above and one ulp below the deciding splat's d, and occluder buffers
   (reverse-Z planes through the cloud with NaN, +inf, -0 and 1.0 pixels): saturated pixels within 4 ulps of the oracle's
   f32 frame, every pixel within blend_cases.frame_bounds of the oracle's depth-tested trace.
4. Buffers whose depths straddle splat depths inside each warp rectangle, frames whose W and H are not multiples of 16,
   and a padded pitch whose padding holds 2.0 (which would hide everything if it were read).
5. Blend-over chains of three clouds over one target and one buffer are byte-identical synchronous, queued or mixed;
   three contexts in flight, each with its own buffer, each produce their own frame.
6. The refusals change nothing; the C++ host (bgs.hpp) and the Python host give identical frames.
7. raster2_kernel<false, true> and raster2_kernel<true, true> with buffers that hide splats (knife, occluder, padded pitch,
   straddling depths) against the oracle, asserting the frame took that path; d bit-exact where the rule's 1e-9 matters
   (h.w ~ 1e-6); splats drawn with h.w in (-1e-9, 0) hidden by a zero buffer; a buffer written on another stream is read
   after that stream's work."""
import ctypes as C

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import blend_cases as BC
import kernel_paths as KP
import test_gpu_blend as TB
from bevy_gaussian_splatting_b200 import abi
from depth_oracle import depth_oracle as D

pytestmark = pytest.mark.gpu


def dev(z):
    import torch

    return torch.from_numpy(np.ascontiguousarray(z, np.float32)).cuda()


def oracle_depths(cloud, view, s, h, ids):
    return D.splat_depth(cloud.position_visibility, view.to_abi(), TB.uniform(s, h), ids)


# ---- 1. the splat depths
LAYOUTS = ("f32", "f16", "f16cov")


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("sort_all", [False, True], ids=["compact", "sort_all"])
@pytest.mark.parametrize("bits", [32, 24, 16])
@pytest.mark.parametrize("gm", [B.GaussianMode.Gaussian3d, B.GaussianMode.Gaussian2d], ids=["3dgs", "2dgs"])
def test_splat_depths_bit_exact(layout, sort_all, bits, gm):
    if layout == "f16cov" and gm != B.GaussianMode.Gaussian3d:
        pytest.skip("a precomputed-covariance cloud is Gaussian3d only")
    cloud = B.random_gaussians_3d_seeded(4000, 11)
    view = B.orbit_view(1, 5, 200, 150)
    s = B.CloudSettings(gaussian_mode=gm, sort_all=sort_all, radix_sort_depth_bits=B.RadixSortDepthBits(bits), global_scale=0.5)
    p = B.GaussianSplattingPlugin(0)
    h = p.add_cloud(cloud, f16=layout == "f16", precompute_covariance=layout == "f16cov")
    zero = dev(np.zeros((view.height, view.width)))
    p.render_view(h, s, view, scene_depth=zero)
    got = p.splat_depths()
    _, ids = p.projected()
    assert len(got) == p.frame_stats().n_visible > 0
    want = oracle_depths(cloud, view, s, h, ids)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


# ---- 2. a zero buffer changes no byte on any path
PATHS = ("r0", "aabb3d", "aabb2d", "r2", "rounds")


def path_case(path):
    cloud = B.random_gaussians_3d_seeded(6000, 21)
    view = B.headless_view(333, 190)   # W, H not multiples of 16
    kw = dict(global_scale=0.5, color_space=B.GaussianColorSpace.LinRec709Display)
    if path == "aabb3d":
        kw["aabb"] = True
    if path == "aabb2d":
        kw.update(aabb=True, gaussian_mode=B.GaussianMode.Gaussian2d)
    if path == "r2":
        kw.update(global_scale=4.0, binning_rounds=False)
    if path == "rounds":
        kw.update(global_scale=4.0, binning_rounds=True)
    if path in ("r0", "aabb3d", "aabb2d"):
        kw["binning_rounds"] = False
    return cloud, view, B.CloudSettings(**kw)


def warm(p, h, s, view, path):
    """r2: the hinted frame after a large-footprint one; the others: a fresh context."""
    if path == "r2":
        p.render_view(h, s, view)
        fs = p.frame_stats()
        assert KP.large_footprint_raster(fs.n_visible, fs.n_pairs)


def hooks(p, rounds):
    fs = p.frame_stats()
    out = [bytes(fs), p.sorted_entries().tobytes()]
    if not rounds:
        out += [p.tile_ranges().tobytes(), p.tile_entries().tobytes()]
    return out


@pytest.mark.parametrize("path", PATHS)
def test_zero_buffer_is_bgs_render_ex(path):
    cloud, view, s = path_case(path)
    zero = dev(np.zeros((view.height, view.width)))
    ps, hs = [], []
    for _ in range(2):
        p = B.GaussianSplattingPlugin(0)
        h = p.add_cloud(cloud)
        warm(p, h, s, view, path)
        ps.append(p); hs.append(h)
    for fmt in ("rgba32f", "rgba16f", "rgba8_srgb"):
        for mode in ("opaque", "premultiplied", "over"):
            for queued in (False, True):
                frames = []
                for k, (p, h) in enumerate(zip(ps, hs)):
                    kw = dict(fmt=fmt, premultiplied=mode == "premultiplied", blend_over=mode == "over", asynchronous=queued)
                    if mode == "over":   # the same seeded target under both
                        tgt = TB.seeded_target(view, 5, fmt)
                        import torch
                        t = torch.from_numpy(tgt.copy()).cuda()
                        p.render_view_to_device(h, s, view, t.data_ptr(), scene_depth=zero if k else None, **kw)
                        if queued:
                            assert p.sync()
                        torch.cuda.synchronize()
                        frames.append(t.cpu().numpy())
                    else:
                        img = p.render_view(h, s, view, scene_depth=zero if k else None, **kw)
                        if queued:
                            assert p.sync()
                        frames.append(img)
                    if path == "rounds":
                        assert p.frame_stats().rounds > 1
                assert frames[0].tobytes() == frames[1].tobytes(), (fmt, mode, queued)
                assert hooks(ps[0], path == "rounds") == hooks(ps[1], path == "rounds"), (fmt, mode, queued)


# ---- 3 / 4. against the oracle's depth-tested walk
def check_frame(p, h, oracle, cloud, view, s, scene_np, scene_arg, name):
    img = p.render_view(h, s, view, fmt="rgba32f", scene_depth=scene_arg)
    _, dc = TB.check_records(p, oracle, cloud, s, view, h)
    u = TB.uniform(s, h)
    trace = D.blend_trace(cloud, view.to_abi(), u, s.to_abi(), scene_np)
    TB.assert_within_bound(name, img, trace, s.aabb, "opaque", dc)
    TB.assert_coverage_map(name, img, D.render_tiles(cloud, view.to_abi(), u, s.to_abi(), scene_np), trace, "opaque")
    return img, trace


@pytest.mark.parametrize("geom", list(BC.GEOMETRIES))
def test_knife_buffers_at_the_deciding_splat(oracle, geom):
    cloud, view, s = BC.saturated_case(geom)
    p = B.GaussianSplattingPlugin(0)
    h = p.add_cloud(cloud)
    u = TB.uniform(s, h)
    tr = D.blend_trace(cloud, view.to_abi(), u, s.to_abi())
    til = oracle.render_tiles(cloud, view.to_abi(), u, s.to_abi(), want_image=False)
    d_rank = D.splat_depth(cloud.position_visibility, view.to_abi(), u, til["rank_to_id"])
    r0 = tr["rank0"]
    has = r0 >= 0
    d0 = np.where(has, d_rank[np.maximum(r0, 0)], np.float32(0))
    inf = np.float32(np.inf)
    for name, z in (("at", d0), ("above", np.where(has, np.nextafter(d0, inf), 0)), ("below", np.where(has, np.nextafter(d0, -inf), 0))):
        z = z.astype(np.float32)
        _, trace = check_frame(p, h, oracle, cloud, view, s, z, dev(z), f"{geom}-knife-{name}")
        first = trace["rank0"]
        if name == "above":
            assert not np.any((first == r0) & has)
        else:
            assert np.array_equal(first[has], r0[has])


def knife_buffers(oracle, cloud, view, s, h):
    """Scene depth exactly at, one ulp above and one ulp below the d of each pixel's first blended splat (0 elsewhere)."""
    u = TB.uniform(s, h)
    tr = D.blend_trace(cloud, view.to_abi(), u, s.to_abi())
    til = oracle.render_tiles(cloud, view.to_abi(), u, s.to_abi(), want_image=False)
    d_rank = D.splat_depth(cloud.position_visibility, view.to_abi(), u, til["rank_to_id"])
    r0 = tr["rank0"]
    has = r0 >= 0
    d0 = np.where(has, d_rank[np.maximum(r0, 0)], np.float32(0)).astype(np.float32)
    inf = np.float32(np.inf)
    return r0, has, {"at": d0, "above": np.where(has, np.nextafter(d0, inf), 0).astype(np.float32),
                     "below": np.where(has, np.nextafter(d0, -inf), 0).astype(np.float32)}


@pytest.mark.parametrize("path", ["r2", "rounds"])
def test_raster2_paths_against_the_oracle(oracle, path):
    """raster2_kernel<false, true> (a hinted large-footprint frame) and raster2_kernel<true, true> (binning rounds, each
    round reading the scene again) with buffers that hide splats: knife buffers, occluders, straddling depths and a padded
    pitch, each held to the oracle's depth-tested walk."""
    cloud, view, s = path_case(path)
    p = B.GaussianSplattingPlugin(0)
    h = p.add_cloud(cloud)
    warm(p, h, s, view, path)
    u = TB.uniform(s, h)

    def took_path():
        fs = p.frame_stats()
        if path == "r2":
            assert fs.rounds == 1 and KP.large_footprint_raster(fs.n_visible, fs.n_pairs)   # this frame's and the next's hint
        else:
            assert fs.rounds > 1

    r0, has, knives = knife_buffers(oracle, cloud, view, s, h)
    for name, z in knives.items():
        _, trace = check_frame(p, h, oracle, cloud, view, s, z, dev(z), f"{path}-knife-{name}")
        took_path()
        first = trace["rank0"]
        if name == "above":
            assert not np.any((first == r0) & has)
        else:
            assert np.array_equal(first[has], r0[has])
    d = D.splat_depth(cloud.position_visibility, view.to_abi(), u, np.arange(len(cloud), dtype=np.uint32))
    rng = np.random.default_rng(11)
    z = occluder(view, d, rng)
    tight, _ = check_frame(p, h, oracle, cloud, view, s, z, dev(z), f"{path}-occluder")
    took_path()
    P = (view.width * 4 + 255) // 256 * 64
    padded = np.full((view.height, P), 2.0, np.float32)
    padded[:, : view.width] = z
    assert p.render_view(h, s, view, fmt="rgba32f", scene_depth=dev(padded)[:, : view.width]).tobytes() == tight.tobytes()
    took_path()
    live = d[np.isfinite(d) & (d > 0)]
    zr = rng.choice(live, view.height * view.width).reshape(view.height, view.width).astype(np.float32)
    check_frame(p, h, oracle, cloud, view, s, zr, dev(zr), f"{path}-straddle")
    took_path()


class RawView:
    """A view whose bgs_view is given as is (the plugin reads only to_abi(), width and height)."""

    def __init__(self, abi_view, width, height):
        self._v, self.width, self.height = abi_view, width, height

    def to_abi(self):
        return self._v


def test_splat_depths_with_a_small_clip_w():
    """A clip matrix scaled by 2^-20: every drawn splat has h.w ~ 1e-6, where the rule's 1e-9 changes d (dropping it would
    change most of these d values); bgs_debug_splat_depths stays bit-exact."""
    base = B.orbit_view(2, 5, 200, 150)
    from bevy_gaussian_splatting_b200.camera import View
    view = View(base.view_from_world, (base.clip_from_view.astype(np.float64) * 2.0 ** -20).astype(np.float32),
                base.world_position, base.width, base.height)
    cloud = B.random_gaussians_3d_seeded(4000, 12)
    s = B.CloudSettings(global_scale=0.5)
    p = B.GaussianSplattingPlugin(0)
    h = p.add_cloud(cloud)
    p.render_view(h, s, view, scene_depth=dev(np.zeros((view.height, view.width))))
    got = p.splat_depths()
    _, ids = p.projected()
    assert len(got) > 100
    want = oracle_depths(cloud, view, s, h, ids)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    va = view.to_abi()
    m = np.array(va.clip_from_world, np.float32)
    pos = cloud.position_visibility[ids]
    hh = [((m[0 + r] * pos[:, 0] + m[4 + r] * pos[:, 1]) + m[8 + r] * pos[:, 2]) + m[12 + r] for r in range(4)]
    assert (hh[3] < 0.03).all()
    no_eps = (hh[2] / hh[3]) / np.float32(1.0)
    assert np.count_nonzero(no_eps.view(np.uint32) != want.view(np.uint32)) > len(want) // 4


def test_negative_w_splats_are_drawn_and_a_zero_buffer_hides_them(oracle):
    """h = (0, 0, 2e-10, -5e-10) for every gaussian: h.w in (-1e-9, 0) passes the frustum test (ndc (0, 0, 0.4)), so
    the splats are drawn at the frame's centre, with pw < 0 and d < 0; a cleared reverse-Z buffer hides them."""
    base = B.headless_view(64, 48)
    va = base.to_abi()
    m = np.zeros(16, np.float32)
    m[14], m[15] = 2e-10, -5e-10
    va.clip_from_world[:] = m.tolist()
    view = RawView(va, base.width, base.height)
    cloud = B.random_gaussians_3d_seeded(50, 13)
    s = B.CloudSettings(global_scale=0.5, color_space=B.GaussianColorSpace.LinRec709Display)
    p = B.GaussianSplattingPlugin(0)
    h = p.add_cloud(cloud)
    plain = p.render_view(h, s, view)
    assert p.frame_stats().n_visible == len(cloud)
    u = TB.uniform(s, h)
    assert np.abs(plain - oracle.render_tiles(cloud, va, u, s.to_abi())["image"]).max() <= 1e-3
    clear = np.zeros_like(plain)
    clear[..., 3] = 1.0
    assert not np.array_equal(plain, clear)
    zero = np.zeros((base.height, base.width), np.float32)
    hidden = p.render_view(h, s, view, scene_depth=dev(zero))
    assert np.array_equal(hidden, clear)
    got = p.splat_depths()
    _, ids = p.projected()
    assert (got < 0).all()
    assert np.array_equal(got.view(np.uint32), D.splat_depth(cloud.position_visibility, va, u, ids).view(np.uint32))
    assert np.array_equal(D.render_tiles(cloud, va, u, s.to_abi(), zero), clear)


def test_producer_stream_is_waited_for():
    """A buffer whose __cuda_array_interface__ names a stream (v3): the frame is ordered after that stream's work."""
    import torch

    view = B.headless_view(96, 64)
    s = B.CloudSettings()
    p = B.GaussianSplattingPlugin(0)
    h = p.add_cloud(B.random_gaussians_3d_seeded(2000, 14))
    side = torch.cuda.Stream()
    z = torch.zeros((view.height, view.width), dtype=torch.float32, device="cuda")
    want = p.render_view(h, s, view, scene_depth=torch.ones_like(z))   # depth 1.0 everywhere: nothing drawn
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)     # keep the producer's stream busy, then write the buffer on it
        z.fill_(1.0)

    class OnSide:
        __cuda_array_interface__ = dict(z.__cuda_array_interface__, version=3, stream=side.cuda_stream)

    got = p.render_view(h, s, view, scene_depth=OnSide())
    assert got.tobytes() == want.tobytes()


def occluder(view, d, rng):
    """Reverse-Z planes and a box through the cloud at splat depths, with NaN, +inf, -0 and 1.0 pixels."""
    H, W = view.height, view.width
    q = np.quantile(d[np.isfinite(d) & (d > 0)], [0.2, 0.5, 0.8]).astype(np.float32)
    z = np.zeros((H, W), np.float32)
    z[:, : W // 2] = q[1]
    z[H // 4: 3 * H // 4, W // 3: 2 * W // 3] = q[2]
    yy, xx = np.mgrid[0:H, 0:W]
    z[(xx + yy) % 7 == 0] = q[0]
    for v in (np.nan, np.inf, -0.0, 1.0):
        idx = rng.choice(H * W, 40, replace=False)
        z.reshape(-1)[idx] = v
    return z


@pytest.mark.parametrize("geom", list(BC.GEOMETRIES))
def test_occluders_padded_pitch_and_straddling_buffers(oracle, geom):
    cloud, view, s = BC.saturated_case(geom, w=250, h=181)
    p = B.GaussianSplattingPlugin(0)
    h = p.add_cloud(cloud)
    u = TB.uniform(s, h)
    d = D.splat_depth(cloud.position_visibility, view.to_abi(), u, np.arange(len(cloud), dtype=np.uint32))
    rng = np.random.default_rng(7)
    z = occluder(view, d, rng)
    tight, _ = check_frame(p, h, oracle, cloud, view, s, z, dev(z), f"{geom}-occluder")
    # the same buffer at a 256-byte-aligned pitch, padding 2.0 (> every d: reading it would hide everything)
    P = (view.width * 4 + 255) // 256 * 64
    padded = np.full((view.height, P), 2.0, np.float32)
    padded[:, : view.width] = z
    t = dev(padded)[:, : view.width]
    assert t.stride(0) == P and t.stride(1) == 1
    assert p.render_view(h, s, view, fmt="rgba32f", scene_depth=t).tobytes() == tight.tobytes()
    # per-pixel depths drawn from the splats' d: every warp rectangle straddles splat depths
    live = d[np.isfinite(d) & (d > 0)]
    zr = rng.choice(live, view.height * view.width).reshape(view.height, view.width).astype(np.float32)
    check_frame(p, h, oracle, cloud, view, s, zr, dev(zr), f"{geom}-straddle")


# ---- 5. compositing chains and contexts in flight
def test_blend_over_chains_and_contexts_in_flight():
    import torch

    view = B.headless_view(240, 136)
    s = B.CloudSettings(global_scale=0.6)
    clouds = [B.random_gaussians_3d_seeded(3000, 30 + k) for k in range(3)]
    zero = np.zeros((view.height, view.width), np.float32)
    zc = clouds[0]
    d = D.splat_depth(zc.position_visibility, view.to_abi(), B.GaussianSplattingPlugin.cloud_uniform(s),
                      np.arange(len(zc), dtype=np.uint32))
    z = zero.copy()
    z[:, : view.width // 2] = np.median(d[np.isfinite(d) & (d > 0)])
    zt = dev(z)
    results = []
    for order in ("sync", "queued", "mixed"):
        p = B.GaussianSplattingPlugin(0)
        hs = [p.add_cloud(c) for c in clouds]
        t = torch.zeros((view.height, view.width, 4), dtype=torch.float32, device="cuda")
        for k, h in enumerate(hs):
            q = order == "queued" or (order == "mixed" and k == 1)
            p.render_view_to_device(h, s, view, t.data_ptr(), fmt="rgba32f", blend_over=True, asynchronous=q, scene_depth=zt)
        assert p.sync()
        torch.cuda.synchronize()
        results.append(t.cpu().numpy().tobytes())
    assert results[0] == results[1] == results[2]
    # three contexts in flight, each its own buffer
    ps = [B.GaussianSplattingPlugin(0) for _ in range(3)]
    hs = [p.add_cloud(clouds[k]) for k, p in enumerate(ps)]
    bufs = [dev(np.roll(z, 40 * k, axis=1)) for k in range(3)]
    want = [p.render_view(h, s, view, scene_depth=b) for p, h, b in zip(ps, hs, bufs)]
    outs = [np.empty_like(w) for w in want]
    for p, h, b, o in zip(ps, hs, bufs, outs):
        p.render_view(h, s, view, scene_depth=b, asynchronous=True, out=o)
    for p in ps:
        assert p.sync()
    for w, o in zip(want, outs):
        assert w.tobytes() == o.tobytes()
    assert want[0].tobytes() != want[1].tobytes()


# ---- 6. refusals
def test_refusals_change_nothing():
    import torch

    view = B.headless_view(96, 64)
    s = B.CloudSettings()
    p = B.GaussianSplattingPlugin(0)
    h = p.add_cloud(B.random_gaussians_3d_seeded(500, 1))
    lib = abi.load()
    u, st, _ = p._call_args(h, s, None)
    v = view.to_abi()
    good = torch.zeros((view.height, view.width + 8), dtype=torch.float32, device="cuda")
    host = np.zeros((view.height, view.width), np.float32)
    cases = [abi.bgs_scene_depth(depth=None, pitch_bytes=4 * view.width),
             abi.bgs_scene_depth(depth=good.data_ptr(), pitch_bytes=4 * view.width + 2),
             abi.bgs_scene_depth(depth=good.data_ptr(), pitch_bytes=4 * view.width - 4),
             abi.bgs_scene_depth(depth=good.data_ptr() + 2, pitch_bytes=4 * view.width + 32),
             abi.bgs_scene_depth(depth=host.ctypes.data, pitch_bytes=4 * view.width)]
    tgt = torch.full((view.height, view.width, 4), 0.25, dtype=torch.float32, device="cuda")
    for zd in cases:
        st_ = lib.bgs_render_depth_test(p._ctx, h._h, C.byref(v), C.byref(u), C.byref(st), None, C.byref(zd),
                                        C.c_void_p(tgt.data_ptr()), abi.BGS_FORMAT_RGBA32F, 1)
        assert st_ == abi.BGS_EINVAL, (zd.depth, zd.pitch_bytes)
        torch.cuda.synchronize()
        assert bool((tgt == 0.25).all())
    # NULL depth: exactly bgs_render_ex
    a = p.render_view(h, s, view)
    out = np.empty_like(a)
    assert lib.bgs_render_depth_test(p._ctx, h._h, C.byref(v), C.byref(u), C.byref(st), None, None, out.ctypes.data,
                                     abi.BGS_FORMAT_RGBA32F, 0) == abi.BGS_OK
    assert a.tobytes() == out.tobytes()


def test_cpp_host_matches_python_host(tmp_path):
    """include/bgs.hpp's render_view_depth_test (examples/headless.cpp --depth-plane) and the Python host give the same
    RGBA8 frame for the same half-frame plane at a 256-byte row pitch."""
    import os
    import subprocess

    import torch

    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
    exe = os.path.join(root, "examples", "headless")
    if not os.path.exists(exe):
        subprocess.run(["make", "-C", os.path.join(root, "examples")], check=True)
    n, w, h, scale, zp = 20000, 320, 200, 0.5, 0.02
    raw, cloud_f = tmp_path / "f.raw", tmp_path / "cloud.bin"
    out = subprocess.run([exe, str(n), str(w), str(h), str(scale), str(tmp_path / "0.ppm"), "--raw", str(raw),
                          "--depth-plane", str(zp), "--dump-cloud", str(cloud_f)], check=True, capture_output=True, text=True).stdout
    assert "rendered=1" in out
    got = np.fromfile(raw, np.uint8).reshape(h, w, 4)
    g = np.fromfile(cloud_f, np.uint8)[8:].view(np.float32)   # the C++ host's cloud, as it uploaded it
    p = B.GaussianSplattingPlugin(0)
    hd = p.add_cloud(B.PlanarGaussian3d(g[: n * 4].reshape(n, 4), g[n * 4: n * 52].reshape(n, 48),
                                        g[n * 52: n * 56].reshape(n, 4), g[n * 56: n * 60].reshape(n, 4)))
    view, s = B.headless_view(w, h), B.CloudSettings(global_scale=scale)
    pitch = (w * 4 + 255) // 256 * 64
    z = torch.zeros((h, pitch), dtype=torch.float32, device="cuda")
    z[:, : w // 2] = float(np.float32(zp))
    want = None
    for _ in range(3):   # (the C++ host renders three frames: the same hints)
        want = p.render_view(hd, s, view, fmt="rgba8_srgb", scene_depth=z[:, :w])
    plain = p.render_view(hd, s, view, fmt="rgba8_srgb")
    assert got.tobytes() == want.tobytes()
    assert got[:, : w // 2].tobytes() != plain[:, : w // 2].tobytes()   # the plane hid something

