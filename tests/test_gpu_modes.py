"""RasterizeMode::Classification and RasterizeMode::OpticalFlow on the GPU (bgs_render_ex, project_modes_kernel).

* Projected records, for every case and geometry of `project_cases` (layouts f32 / f16 / f16 covariance, identity and
  general models, both colour spaces, every draw mode): geometry, bboxes, opacity and the drawn decision are those of the
  Color-mode records of the same frame, bit for bit.  Classification colours are `modes_oracle.class_colour` of the
  GPU's own Color colours bit for bit, and within half of `project_cases.colour_bound` (+ 1 ulp for the mix's last
  rounding) of the oracle's; OpticalFlow colours equal the oracle's bit for bit (the atan2 is the shared f64 series).
* Identities, byte for byte: Classification with every vis < 2 is the Color frame; OpticalFlow with an unmoved camera
  colours every splat (1, 1, 1).
* Whole frames against oracle/'s tile_mode walk: the oracle renders a proxy cloud whose Color-mode colours (linear
  colour space, SH degree 0) stand for the mode's colours; `blend_cases.frame_bounds` with dc = the largest measured
  difference between the GPU's mode colours and the proxy's oracle colours bounds every pixel, in RGBA32F, RGBA16F and
  RGBA8, synchronous, queued, chunked and blended over a target.  Labels edited between queued frames reach each frame.
* Refusals change nothing and launch nothing; bgs_render_ex(..., NULL, ...) is bgs_render for the four other modes.
"""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import blend_cases as BC
import modes_cases as MC
import project_cases as PC
from bevy_gaussian_splatting_b200 import abi
from modes_oracle import modes_oracle as MO

pytestmark = pytest.mark.gpu

f32 = np.float32
RM = B.RasterizeMode
C0 = f32(0.28209479177387814)


@pytest.fixture(scope="module")
def plugin():
    p = B.GaussianSplattingPlugin(0)
    yield p
    p.destroy()


@pytest.fixture(scope="module")
def cases(oracle):
    return {c.name: c for c in PC.all_cases(oracle)}


def moved(view, dx=0.03, dy=-0.02, dz=0.05):
    """The previous frame's view: the same camera, offset."""
    eye = np.asarray(view.world_position, np.float64)
    return B.perspective_view(tuple(eye + (dx, dy, dz)), tuple(eye + (dx, dy, dz - 1.0)), view.width, view.height)


def extras_of(s, prev=None, dt=None):
    ex = abi.bgs_render_extras(num_classes=int(s.num_classes))
    if prev is not None:
        ex.previous_clip_from_world[:] = prev.to_abi().clip_from_world[:]
        ex.delta_time = dt
    return ex


def labels_for(n, num_classes, seed):
    """A mix of unlabelled (< 2) and labelled gaussians, class boundaries, fractional labels and the wrap."""
    rng = np.random.default_rng(seed)
    pool = MC.class_labels(num_classes)
    pool = pool[np.isfinite(pool) | (pool == -np.inf)]
    return rng.choice(pool, n).astype(f32)


def geometry_equal(rec, ref):
    """Every record's centre, uv rows, bbox and opacity equal bit for bit (all records, drawn or not)."""
    cols = [0, 1, 2, 3, 4, 5, 6, 7, 11]
    return np.array_equal(rec[:, cols].view(np.uint32), ref[:, cols].view(np.uint32))


def drawn_of(rec):
    bb = rec[:, 6:8].view(np.uint32)
    return ((bb[:, 0] & 0xFFFF) <= (bb[:, 0] >> 16)) & ((bb[:, 1] & 0xFFFF) <= (bb[:, 1] >> 16))


def records(plugin, h, s, view, transform=None, prev=None, dt=None):
    plugin.render_view(h, s, view, transform=transform, previous_view=prev, delta_time=dt)
    return plugin.projected()


# ---------------------------------------------------------------------------------------------------------------------
# projected records, every project_cases case

def _params():
    return [(name, g) for name, geoms in PC.case_index() if not name.startswith("sh_") for g in geoms]


PARAMS = _params()


@pytest.mark.parametrize("name,geom", PARAMS, ids=[f"{n}-{g}" for n, g in PARAMS])
def test_records_vs_color_and_oracle(plugin, oracle, cases, name, geom):
    case = cases[name]
    oc = case.oracle_cloud()
    h = plugin.add_cloud(case.cloud, f16=case.layout == "f16", precompute_covariance=case.layout == "cov")
    try:
        for k, num_classes in enumerate(MC.NUM_CLASSES):
            s = PC.settings(geom, **{**case.settings, "num_classes": num_classes})
            vis = labels_for(len(oc), num_classes, k)
            if s.draw_mode == B.DrawMode.All:
                plugin.set_visibility(h, vis)
            else:
                vis = plugin.visibility(h)   # the case's own selection decides what is drawn
            col, ids = records(plugin, h, dataclasses.replace(s, rasterize_mode=RM.Color), case.view, case.transform)
            cls, ids2 = records(plugin, h, dataclasses.replace(s, rasterize_mode=RM.Classification), case.view, case.transform)
            assert np.array_equal(ids, ids2)
            assert geometry_equal(cls, col), "Classification geometry differs from Color's"
            drawn = drawn_of(col)
            u = plugin.cloud_uniform(s, case.transform, h.aabb)
            lit = (s.draw_mode == B.DrawMode.HighlightSelected) & (vis[ids] > 0.5)
            own = MO.class_colour(col[:, 8:11], vis[ids], num_classes)
            own[lit] = MO.HIGHLIGHT
            ok = MC.same_bits(cls[drawn, 8:11], own[drawn])
            assert ok.all(), f"class colour of gaussian {ids[drawn][np.argwhere(~ok)[0][0]]} is not mix(sh, hue) of its Color colour"
            if drawn.any():
                sa = dataclasses.replace(s, rasterize_mode=RM.Classification).to_abi()
                sa.reserved = 1 if case.layout == "cov" else 0
                pv = oc.position_visibility.copy()
                pv[:, 3] = vis
                ocl = B.PlanarGaussian3d(pv, oc.spherical_harmonic, oc.rotation, oc.scale_opacity)
                orec = MO.project_ex(oracle, ocl, case.view.to_abi(), u, sa, extras_of(s), ids)
                want = np.stack([orec[c] for c in "rgb"], 1)[drawn]
                bound = PC.colour_bound(oc, case.view, case.model, int(s.color_space), ids[drawn])
                hue = (vis[ids][drawn] >= 2) | np.isnan(vis[ids][drawn])
                bound = np.where(hue[:, None], 0.5 * bound + np.spacing(np.abs(want).astype(f32)), bound)
                bound[lit[drawn]] = 0.0
                assert PC.colours_agree(cls[drawn, 8:11], want, bound).all(), "class colour outside the derived bound"
        # OpticalFlow: a moved camera, and an unmoved one
        s = PC.settings(geom, **case.settings)
        sa = dataclasses.replace(s, rasterize_mode=RM.OpticalFlow).to_abi()
        sa.reserved = 1 if case.layout == "cov" else 0
        u = plugin.cloud_uniform(s, case.transform, h.aabb)
        col, ids = records(plugin, h, dataclasses.replace(s, rasterize_mode=RM.Color), case.view, case.transform)
        drawn = drawn_of(col)
        vis = plugin.visibility(h)
        lit = (s.draw_mode == B.DrawMode.HighlightSelected) & (vis[ids] > 0.5)
        for prev, dt in ((moved(case.view), 1 / 60), (moved(case.view, 0.5, 0.2, -0.3), 0.25), (case.view, 1 / 30)):
            fl, ids2 = records(plugin, h, dataclasses.replace(s, rasterize_mode=RM.OpticalFlow), case.view, case.transform, prev, dt)
            assert np.array_equal(ids, ids2) and geometry_equal(fl, col), "OpticalFlow geometry differs from Color's"
            pv = oc.position_visibility.copy()
            pv[:, 3] = vis
            ocl = B.PlanarGaussian3d(pv, oc.spherical_harmonic, oc.rotation, oc.scale_opacity)
            orec = MO.project_ex(oracle, ocl, case.view.to_abi(), u, sa, extras_of(s, prev, dt), ids)
            want = np.stack([orec[c] for c in "rgb"], 1)
            ok = MC.same_bits(fl[drawn, 8:11], want[drawn])
            assert ok.all(), f"flow colour of gaussian {ids[drawn][np.argwhere(~ok)[0][0]]}: {fl[drawn][np.argwhere(~ok)[0][0], 8:11]} vs {want[drawn][np.argwhere(~ok)[0][0]]}"
            if prev is case.view:
                assert (fl[drawn & ~lit, 8:11] == 1.0).all(), "an unmoved camera must give white splats"
    finally:
        h.destroy()


@pytest.mark.parametrize("num_classes", MC.NUM_CLASSES)
def test_every_label_bit_exact(plugin, num_classes):
    """Every label of `modes_cases.class_labels` (NaN and +-inf included) on a few hundred drawn gaussians each, both colour
    spaces: the Classification colour is mix(sh, hue) of the same frame's Color colour, bit for bit.  (The remainder's
    x - 6 trunc(x / 6) and fmodf part only at labels like 1e30, which this covers.)"""
    cloud = B.random_gaussians_3d_seeded(40000, 8)
    view = B.headless_view(320, 200)
    pool = MC.class_labels(num_classes)
    vis = np.resize(pool, len(cloud)).astype(f32)
    h = plugin.add_cloud(cloud)
    try:
        plugin.set_visibility(h, vis)
        for cs in B.GaussianColorSpace:
            s = B.CloudSettings(num_classes=num_classes, color_space=cs)
            col, ids = records(plugin, h, s, view)
            cls, _ = records(plugin, h, dataclasses.replace(s, rasterize_mode=RM.Classification), view)
            drawn = drawn_of(col)
            assert geometry_equal(cls, col)
            seen = set(vis[ids[drawn]].view(np.uint32).tolist())
            assert seen >= set(pool.view(np.uint32).tolist()) - {f32(np.nan).view(np.uint32), f32(-np.nan).view(np.uint32)}
            ok = MC.same_bits(cls[drawn, 8:11], MO.class_colour(col[drawn, 8:11], vis[ids[drawn]], num_classes))
            assert ok.all(), f"label {vis[ids[drawn]][np.argwhere(~ok)[0][0]]!r}"
    finally:
        h.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# identities

def test_classification_below_two_is_the_color_frame(plugin):
    cloud = B.random_gaussians_3d_seeded(30000, 3)
    view = B.headless_view(320, 200)
    h = plugin.add_cloud(cloud)
    try:
        vis = np.random.default_rng(0).choice(np.array([-np.inf, 0.0, 0.5, 1.0, 1.9999999], f32), len(cloud))
        plugin.set_visibility(h, vis)
        for fmt in ("rgba32f", "rgba16f", "rgba8_srgb"):
            for geom in BC.GEOMETRIES:
                s = BC.settings_for(geom, False, num_classes=3)
                a = plugin.render_view(h, s, view, fmt=fmt)
                b = plugin.render_view(h, dataclasses.replace(s, rasterize_mode=RM.Classification), view, fmt=fmt)
                assert a.tobytes() == b.tobytes(), (fmt, geom)
    finally:
        h.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# whole frames against the oracle's tile_mode walk

def proxy_cloud(cloud, ids, rgb):
    """`cloud` with SH degree 0 set so that Color mode in the linear colour space gives (about) rgb for ids."""
    sh = np.zeros_like(cloud.spherical_harmonic)
    sh[ids, 0:3] = (rgb - f32(0.5)) / C0
    return B.PlanarGaussian3d(cloud.position_visibility, sh, cloud.rotation, cloud.scale_opacity)


def render_dev(p, h, s, view, out_mode, fmt="rgba32f", dst=None, prev=None, dt=None):
    import torch

    code, dtype, _ = B.GaussianSplattingPlugin.FORMATS[fmt]
    tdt = {np.float32: torch.float32, np.float16: torch.float16, np.uint8: torch.uint8}[dtype]
    tgt = torch.zeros((view.height, view.width, 4), dtype=tdt, device="cuda")
    if dst is not None:
        tgt.copy_(torch.from_numpy(np.ascontiguousarray(dst)))
    torch.cuda.synchronize()
    p.render_view_to_device(h, s, view, tgt.data_ptr(), fmt=fmt, premultiplied=out_mode == "premultiplied",
                            blend_over=out_mode == "over", previous_view=prev, delta_time=dt)
    torch.cuda.synchronize()
    return tgt.cpu().numpy()


def frame_reference(oracle, p, h, cloud, s, view, vis, prev=None, dt=None):
    """(trace of the proxy, dc, records) for the frame p last rendered in s's mode."""
    rec, ids = p.projected()
    drawn = drawn_of(rec)
    pv = cloud.position_visibility.copy()
    pv[:, 3] = vis
    proxy = proxy_cloud(B.PlanarGaussian3d(pv, cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity), ids, rec[:, 8:11])
    sl = dataclasses.replace(s, rasterize_mode=RM.Color, color_space=B.GaussianColorSpace.LinRec709Display)
    u = p.cloud_uniform(sl, None, h.aabb)
    orec = oracle.project(proxy, view.to_abi(), u, sl.to_abi(), ids)
    want = np.stack([orec[c] for c in "rgb"], 1)
    dc = float(np.abs(rec[drawn, 8:11].astype(np.float64) - want[drawn]).max()) if drawn.any() else 0.0
    trace = oracle.blend_trace(proxy, view.to_abi(), u, sl.to_abi())
    return trace, dc


def check_frame(name, got, trace, aabb, out_mode, dc, dst=None):
    want = BC.expected_frame(trace, out_mode, dst)
    bound, _ = BC.frame_bounds(trace, aabb, out_mode, dc, dst)
    err = np.abs(got.astype(np.float64) - want)
    bad = np.argwhere(err > bound)
    assert not len(bad), f"{name}: {len(bad)} channels outside the bound, first {tuple(bad[0])}: err {err[tuple(bad[0])]:.3g} > {bound[tuple(bad[0])]:.3g}"


FRAME_PARAMS = [(m, g) for m in ("classification", "flow") for g in BC.GEOMETRIES]


@pytest.mark.parametrize("mode,geom", FRAME_PARAMS)
def test_frames_vs_oracle(oracle, mode, geom):
    from test_gpu_blend import assert_quantised, seeded_target

    aabb = BC.GEOMETRIES[geom][1]
    cloud = B.random_gaussians_3d_seeded(20000, 5)
    view = B.headless_view(256, 160)
    vis = labels_for(len(cloud), 3, 1)
    prev, dt = (moved(view), 1 / 60) if mode == "flow" else (None, None)
    rm = RM.Classification if mode == "classification" else RM.OpticalFlow
    s = BC.settings_for(geom, False, rasterize_mode=rm, num_classes=3)
    p = B.GaussianSplattingPlugin(0)
    try:
        h = p.add_cloud(cloud)
        p.set_visibility(h, vis)
        base = p.render_view(h, s, view, previous_view=prev, delta_time=dt)
        trace, dc = frame_reference(oracle, p, h, cloud, s, view, vis, prev, dt)
        check_frame(f"{mode}/{geom}/sync", base, trace, aabb, "opaque", dc)
        # queued and chunked frames are the same bytes
        out = np.empty_like(base)
        p.render_view(h, s, view, out=out, asynchronous=True, previous_view=prev, delta_time=dt)
        assert p.sync()
        assert out.tobytes() == base.tobytes(), "queued frame differs"
        if not aabb:
            ch = p.render_view(h, dataclasses.replace(s, binning_rounds=True), view, previous_view=prev, delta_time=dt)
            assert p.frame_stats().rounds > 1
            assert ch.tobytes() == base.tobytes(), "chunked frame differs"
        for out_mode in ("opaque", "premultiplied", "over"):
            dst = seeded_target(view, 7) if out_mode == "over" else None
            got = render_dev(p, h, s, view, out_mode, dst=dst, prev=prev, dt=dt)
            check_frame(f"{mode}/{geom}/{out_mode}", got, trace, aabb, out_mode, dc, dst)
            for fmt in ("rgba16f", "rgba8_srgb"):
                dq = seeded_target(view, 7, fmt) if out_mode == "over" else None
                q = render_dev(p, h, s, view, out_mode, fmt, dst=dq, prev=prev, dt=dt)
                assert_quantised(q, trace, aabb, out_mode, fmt, dc, dst=dq)
        h.destroy()
    finally:
        p.destroy()


def test_labels_edited_between_queued_frames(plugin):
    cloud = B.random_gaussians_3d_seeded(20000, 6)
    view = B.headless_view(256, 160)
    s = BC.settings_for("obb3d", False, rasterize_mode=RM.Classification, num_classes=4)
    h = plugin.add_cloud(cloud)
    try:
        labs = [labels_for(len(cloud), 4, k) for k in range(3)]
        want = []
        for v in labs:
            plugin.set_visibility(h, v)
            want.append(plugin.render_view(h, s, view))
        outs = [np.empty_like(want[0]) for _ in labs]
        for v, o in zip(labs, outs):
            plugin.set_visibility(h, v)
            plugin.render_view(h, s, view, out=o, asynchronous=True)
        assert plugin.sync()
        for k, (o, w) in enumerate(zip(outs, want)):
            assert o.tobytes() == w.tobytes(), f"queued frame {k} does not show its own labels"
        assert want[0].tobytes() != want[1].tobytes()
    finally:
        h.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# refusals, and bgs_render_ex(..., NULL, ...) == bgs_render

def _call(p, h, s, view, ex, out):
    v, u = view.to_abi(), p.cloud_uniform(B.CloudSettings(), None, h.aabb)
    sa = s.to_abi() if not isinstance(s, abi.bgs_settings) else s
    return p._lib.bgs_render_ex(p._ctx, h._h, C.byref(v), C.byref(u), C.byref(sa), None if ex is None else C.byref(ex),
                                out.ctypes.data_as(C.c_void_p), abi.BGS_FORMAT_RGBA32F, 0)


def test_refusals_change_nothing(plugin):
    cloud = B.random_gaussians_3d_seeded(5000, 2)
    view = B.headless_view(128, 96)
    h = plugin.add_cloud(cloud)
    try:
        s = B.CloudSettings(num_classes=3)
        out = plugin.render_view(h, s, view)
        launches, before = plugin.last_launch_count, out.copy()
        good = extras_of(s, moved(view), 1 / 60)
        bad = []
        bad.append((dataclasses.replace(s, rasterize_mode=RM.Classification), abi.bgs_render_extras(num_classes=0)))
        bad.append((dataclasses.replace(s, rasterize_mode=RM.OpticalFlow), None))
        for dt in (0.0, -1.0, float("inf"), float("nan"), -0.0):
            e = extras_of(s, moved(view), 1.0)
            e.delta_time = dt
            bad.append((dataclasses.replace(s, rasterize_mode=RM.OpticalFlow), e))
        for i, x in ((0, float("nan")), (15, float("inf")), (5, float("-inf"))):
            e = extras_of(s, moved(view), 1.0)
            e.previous_clip_from_world[i] = x
            bad.append((dataclasses.replace(s, rasterize_mode=RM.OpticalFlow), e))
        velocity = s.to_abi()
        velocity.rasterize_mode = 6
        bad.append((velocity, good))
        for st, ex in bad:
            assert _call(plugin, h, st, view, ex, out) == abi.BGS_EINVAL
            assert plugin.last_launch_count == launches and out.tobytes() == before.tobytes()
        for rm in (RM.Classification, RM.OpticalFlow):
            with pytest.raises(abi.BgsError):
                plugin.render_view_aux(h, dataclasses.replace(s, rasterize_mode=rm), view)
            assert plugin.last_launch_count == launches
        # a refused call leaves the last frame's hooks as they were
        assert plugin.frame_stats().width == 128
        # bgs_render_ex(..., NULL, ...) is bgs_render for the four other modes
        for rm in (RM.Color, RM.Depth, RM.Normal, RM.Position):
            st = dataclasses.replace(s, rasterize_mode=rm)
            a = np.empty_like(out)
            v, u, sa = view.to_abi(), plugin.cloud_uniform(st, None, h.aabb), st.to_abi()
            plugin._check(plugin._lib.bgs_render(plugin._ctx, h._h, C.byref(v), C.byref(u), C.byref(sa), a.ctypes.data_as(C.c_void_p),
                                                 abi.BGS_FORMAT_RGBA32F, 0))
            na = plugin.last_launch_count
            b = np.empty_like(out)
            assert _call(plugin, h, st, view, None, b) == abi.BGS_OK
            assert a.tobytes() == b.tobytes() and plugin.last_launch_count == na, rm
            c = np.empty_like(out)
            assert _call(plugin, h, st, view, good, c) == abi.BGS_OK       # extras are ignored by these modes
            assert a.tobytes() == c.tobytes(), rm
    finally:
        h.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# at scale

@pytest.mark.parametrize("mode", ["classification", "flow"])
def test_6m_f16_frame(oracle, mode):
    n = 6_000_000
    cloud = B.random_gaussians_3d_seeded(n, 11)
    oc = cloud.rounded_to_f16()
    view = B.headless_view(1920, 1080)
    prev, dt = (moved(view), 1 / 60) if mode == "flow" else (None, None)
    rm = RM.Classification if mode == "classification" else RM.OpticalFlow
    s = B.CloudSettings(rasterize_mode=rm, num_classes=7, global_scale=0.25, binning_rounds=False)
    vis = labels_for(n, 7, 2)
    p = B.GaussianSplattingPlugin(0)
    try:
        h = p.add_cloud(cloud, f16=True)
        p.set_visibility(h, vis)
        img = p.render_view(h, s, view, previous_view=prev, delta_time=dt)
        sc = dataclasses.replace(s, rasterize_mode=RM.Color)
        u = p.cloud_uniform(sc, None, h.aabb)
        keys = oracle.keygen(oc.position_visibility, view.to_abi(), u, 32)
        sk, si = oracle.radix_sort(keys, 32)
        got = p.sorted_entries()
        assert np.array_equal(got[:, 0], sk) and np.array_equal(got[:, 1], si), "sort order not bit-exact"
        til = oracle.render_tiles(oc, view.to_abi(), u, sc.to_abi(), want_image=False)
        assert np.array_equal(p.tile_ranges(), til["tile_ranges"]), "tile ranges not bit-exact"
        trace, dc = frame_reference(oracle, p, h, oc, s, view, vis, prev, dt)
        check_frame(f"6M {mode}", img, trace, False, "opaque", dc)
        h.destroy()
    finally:
        p.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# the C++ host

@pytest.mark.parametrize("mode", ["classification", "optical-flow"])
def test_cpp_host_matches_python_host(plugin, tmp_path, mode):
    import os
    import subprocess

    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
    exe = os.path.join(root, "examples", "headless")
    if not os.path.exists(exe):
        subprocess.run(["make", "-C", os.path.join(root, "examples")], check=True)
    n, w, h, scale = 20000, 320, 200, 0.5
    raw, cloud_f = tmp_path / "f.raw", tmp_path / "cloud.bin"
    out = subprocess.run([exe, str(n), str(w), str(h), str(scale), str(tmp_path / "0.ppm"), "--raw", str(raw), "--rasterize", mode,
                          "--num-classes", "5", "--prev-view", "0.1,-0.05,0.2", "--dump-cloud", str(cloud_f)],
                         check=True, capture_output=True, text=True).stdout
    assert "rendered=1" in out
    got = np.fromfile(raw, np.uint8).reshape(h, w, 4)
    g = np.fromfile(cloud_f, np.uint8)[8:].view(f32)
    hd = plugin.add_cloud(B.PlanarGaussian3d(g[: n * 4].reshape(n, 4), g[n * 4: n * 52].reshape(n, 48),
                                             g[n * 52: n * 56].reshape(n, 4), g[n * 56: n * 60].reshape(n, 4)))
    try:
        view = B.headless_view(w, h)
        if mode == "classification":
            s = B.CloudSettings(global_scale=scale, rasterize_mode=RM.Classification, num_classes=5)
            plugin.set_visibility(hd, (2.0 + np.arange(n) % 5).astype(f32))
            want = plugin.render_view(hd, s, view, fmt="rgba8_srgb")
        else:
            words = next(line for line in out.splitlines() if line.startswith("prev_clip:")).split()[1:]
            prev_clip = np.array([int(x, 16) for x in words], np.uint32).view(f32)
            s = B.CloudSettings(global_scale=scale, rasterize_mode=RM.OpticalFlow)
            ex = abi.bgs_render_extras(num_classes=1, delta_time=f32(1.0 / 60.0))
            ex.previous_clip_from_world[:] = prev_clip.tolist()
            want = np.empty((h, w, 4), np.uint8)
            v, u, sa = view.to_abi(), plugin.cloud_uniform(s, None, hd.aabb), s.to_abi()
            plugin._check(plugin._lib.bgs_render_ex(plugin._ctx, hd._h, C.byref(v), C.byref(u), C.byref(sa), C.byref(ex),
                                                    want.ctypes.data_as(C.c_void_p), abi.BGS_FORMAT_RGBA8_SRGB, 0))
        assert got.tobytes() == want.tobytes()
    finally:
        hd.destroy()
