"""bgs_render_shutter on the H100.  One sample is bgs_render_entities_ex byte for byte, hooks and launch count included,
for every mix the views tests use, in every format and output mode, into host and device targets, with and without a
depth buffer.  2, 4 and 16 equal samples give that frame byte for byte.  Samples that differ in camera, entity transform
and Gaussian4d time give the pairwise mean of their bgs_render_entities_ex frames: bit for bit in premultiplied rgb,
within the rule's rounding in alpha and the encoders' bands in RGBA16F and RGBA8.  The hooks restricted to a sample are
its own, and the launch count is the views frame's plus one.  The frame matches the mean of the entity oracle's frames.
Queued frames, the pair-list overflow and the refusals behave as include/bgs.h rules, and the C++ host's frame is the
Python host's."""
import ctypes as C
import dataclasses
import os
import subprocess

import numpy as np
import pytest
import torch

import bevy_gaussian_splatting_b200 as B
import entity_cases as E
import output_cases as O
import shutter_cases as SH
import views_cases as V
import views_scale_cases as VS
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import entity_settings
from entity_oracle import entity_oracle as EO

pytestmark = pytest.mark.gpu

PIXEL_TOL = 1e-3
M = B.RasterizeMode
FORMATS = {"f32": (np.float32, torch.float32, abi.BGS_FORMAT_RGBA32F), "f16": (np.float16, torch.float16, abi.BGS_FORMAT_RGBA16F),
           "u8": (np.uint8, torch.uint8, abi.BGS_FORMAT_RGBA8_SRGB)}
OUT_NAME = {"f32": "rgba32f", "f16": "rgba16f", "u8": "rgba8_srgb"}
PREMUL, OVER, ASYNC = abi.BGS_FLAG_PREMULTIPLIED_OUT, abi.BGS_FLAG_BLEND_OVER_TARGET, abi.BGS_FLAG_ASYNC


def _ok(p, rc):
    assert rc == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)


def _depth(view, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand((view.height, view.width), generator=g, device="cuda") * 0.04


def _noise(view, fmt, seed):
    rng = np.random.default_rng(seed)
    if fmt == "u8":
        return rng.integers(0, 256, (view.height, view.width, 4), dtype=np.uint8)
    return rng.random((view.height, view.width, 4), dtype=np.float32).astype(FORMATS[fmt][0])


def _target(view, fmt, device, fill=None):
    npd, tod, _ = FORMATS[fmt]
    if device:
        t = torch.empty((view.height, view.width, 4), dtype=tod, device="cuda")
        if fill is not None:
            t.copy_(torch.from_numpy(fill))
        return t
    return np.empty((view.height, view.width, 4), npd) if fill is None else fill.copy()


def _addr(t):
    return t.data_ptr() if isinstance(t, torch.Tensor) else t.ctypes.data


def _host(t):
    if isinstance(t, torch.Tensor):
        torch.cuda.synchronize()
        return t.cpu().numpy()
    return t


def _hooks(p, depth_tested):
    fs = p.frame_stats()
    rec, ids = p.projected()
    got = dict(stats=fs, sorted=p.sorted_entries(), records=rec, ids=ids, ranges=p.tile_ranges(), entries=p.tile_entries())
    got["splat_depths"] = p.splat_depths() if depth_tested else None
    return got


def _same_hooks(got, want):
    assert bytes(got["stats"]) == bytes(want["stats"])
    for key in ("sorted", "records", "ids", "ranges", "entries", "splat_depths"):
        assert (got[key] is None) == (want[key] is None), key
        if got[key] is not None:
            assert got[key].tobytes() == want[key].tobytes(), key


class Shutter:
    """One mix's clouds on a context and the s samples of a shutter over them (shutter_cases): the arguments of its
    bgs_render_shutter call and of each sample's bgs_render_entities_ex call."""

    def __init__(self, p, mix, s, moving=True, scale=None, views=None):
        self.p = p
        listed, self.bits, self.frame_box = V.entities(mix)
        if scale is not None:
            listed = [(c, lay, tr, dataclasses.replace(st, global_scale=scale)) for c, lay, tr, st in listed]
        up = {}
        self.handles = []
        for cloud, layout, _, _ in listed:
            if id(cloud) not in up:
                up[id(cloud)] = p.add_cloud(cloud, f16=layout in ("f16", "cov"), precompute_covariance=layout == "cov")
            self.handles.append(up[id(cloud)])
        self.samples = SH.sample_entities(listed, s, moving)
        self.views = views if views is not None else SH.sample_views(s, moving)
        self.sts = [st for _, _, _, st in listed]
        self.unis = [[p.cloud_uniform(st, tr, h.aabb) for h, (_, _, tr, st) in zip(self.handles, smp)] for smp in self.samples]

    @property
    def s(self):
        return len(self.samples)

    def oracle(self, i):
        return [E.oracle_entry(c, lay, u, st) for (c, lay, _, st), u in zip(self.samples[i], self.unis[i])]

    def plugin_samples(self):
        return [[(h, st, tr if tr is not None else B.CloudTransform()) for h, (_, _, tr, st) in zip(self.handles, smp)]
                for smp in self.samples]

    def common(self, flags=0, ents=None):
        k = len(self.handles)
        s = self.sts[0].to_abi()
        s.flags = (s.flags & ~abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX) | flags | (abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX if self.frame_box else 0)
        return ((C.c_void_p * k)(*[h._h.value for h in self.handles]),
                (abi.bgs_entity_settings * k)(*(ents or [entity_settings(st) for st in self.sts])), (C.c_uint32 * k)(*self.bits), k, s)

    def shutter(self, out, fmt, flags=0, depths=None, device=False, ents=None, unis=None, views=None, target=-1):
        clouds, es, bits, k, s = self.common(flags, ents)
        unis = self.unis if unis is None else unis
        views = self.views if views is None else views
        n = len(views)
        flat = [u for smp in unis for u in smp]
        us = (abi.bgs_cloud_uniform * max(len(flat), 1))(*flat)
        vs = (abi.bgs_view * max(n, 1))(*[v.to_abi() for v in views])
        zds = None if depths is None else (abi.bgs_scene_depth * n)(
            *[abi.bgs_scene_depth(depth=d.data_ptr(), pitch_bytes=4 * v.width) for d, v in zip(depths, views)])
        return self.p._lib.bgs_render_shutter(self.p._ctx, clouds, us, es, bits, k, vs, n, C.byref(s), zds,
                                              _addr(out) if target == -1 else target, FORMATS[fmt][2], int(device))

    def ex(self, i, out, fmt, flags=0, depth=None, device=False):
        clouds, es, bits, k, s = self.common(flags)
        view = self.views[i]
        zd = None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * view.width)
        return self.p._lib.bgs_render_entities_ex(self.p._ctx, clouds, (abi.bgs_cloud_uniform * k)(*self.unis[i]), es, bits, k,
                                                  C.byref(view.to_abi()), C.byref(s), None, None if zd is None else C.byref(zd),
                                                  _addr(out), FORMATS[fmt][2], int(device))

    def views_frame(self, fmt="f32"):
        """bgs_render_views of sample 0's entities from the s views, into host frames"""
        clouds, es, bits, k, s = self.common()
        n = len(self.views)
        outs = [_target(v, fmt, False) for v in self.views]
        return self.p._lib.bgs_render_views(self.p._ctx, clouds, (abi.bgs_cloud_uniform * k)(*self.unis[0]), es, bits, k,
                                            (abi.bgs_view * n)(*[v.to_abi() for v in self.views]), n, C.byref(s), None,
                                            (C.c_void_p * n)(*[o.ctypes.data for o in outs]), FORMATS[fmt][2], 0)


def _runs(view, depth):
    """(fmt, device, flags, depth, seed fill or None) of every output variant: all formats and both targets opaque and
    premultiplied, and blend-over into device targets seeded with noise and into host targets (over the context's last
    frame, which the caller seeds); the depth buffer on some of them"""
    runs = [(fmt, device, flags, depth if fmt != "f16" else None, None)
            for fmt in FORMATS for device in (False, True) for flags in (0, PREMUL)]
    runs += [(fmt, True, OVER, depth, _noise(view, fmt, 11)) for fmt in FORMATS]
    runs += [(fmt, False, OVER, None, None) for fmt in FORMATS]
    return runs


def _render_pair(p, sc, fmt, device, flags, depth, fill, call_got, call_want):
    """(got, want) host copies of two calls into fresh targets of one output variant (host blend-over: each over the
    same seeded last frame)"""
    view = sc.views[0]
    frames = []
    for call in (call_got, call_want):
        if flags & OVER and not device:
            _ok(p, sc.ex(0, _target(view, fmt, False), fmt, 0))   # (the library frame both blend over)
        out = _target(view, fmt, device, fill)
        _ok(p, call(out))
        frames.append((_host(out).copy(), p.last_launch_count))
    return frames


# ---- 1. one sample is bgs_render_entities_ex

@pytest.mark.parametrize("mix", list(V.MIXES))
@pytest.mark.parametrize("with_depth", [False, True])
def test_one_sample_is_entities_ex(mix, with_depth):
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Shutter(p, mix, 1)
        view = sc.views[0]
        depth = _depth(view, 3) if with_depth else None
        for fmt, device, flags, d, fill in _runs(view, depth):
            dd = None if d is None else [d]
            out = _target(view, fmt, device, fill)
            if flags & OVER and not device:
                _ok(p, sc.ex(0, _target(view, fmt, False), fmt, 0))
            _ok(p, sc.shutter(out, fmt, flags, dd, device))
            got, gl, gh = _host(out).copy(), p.last_launch_count, _hooks(p, d is not None)
            want = _target(view, fmt, device, fill)
            if flags & OVER and not device:
                _ok(p, sc.ex(0, _target(view, fmt, False), fmt, 0))
            _ok(p, sc.ex(0, want, fmt, flags, d, device))
            assert got.tobytes() == _host(want).tobytes(), (fmt, device, flags)
            assert gl == p.last_launch_count
            _same_hooks(gh, _hooks(p, d is not None))
    finally:
        p.destroy()


# ---- 2. equal samples are the one-sample frame

@pytest.mark.parametrize("mix,s", [("mixed_conic", 2), ("mixed_conic", 4), ("mixed_conic", 16), ("mixed", 2), ("mixed", 4),
                                   ("surfel", 16), ("quad_box", 4)])
def test_equal_samples_are_the_one_sample_frame(mix, s):
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Shutter(p, mix, s, moving=False)
        view = sc.views[0]
        depth = _depth(view, 5)
        for fmt, device, flags, d, fill in _runs(view, depth):
            (got, _), (want, _) = _render_pair(p, sc, fmt, device, flags, d, fill,
                                               lambda o: sc.shutter(o, fmt, flags, None if d is None else [d] * s, device),
                                               lambda o: sc.ex(0, o, fmt, flags, d, device))
            assert got.tobytes() == want.tobytes(), (fmt, device, flags, d is not None)
    finally:
        p.destroy()


# ---- 3. samples that differ: the pairwise mean of their frames

@pytest.mark.parametrize("s", [3, 5, 8])
def test_moving_samples_are_the_mean_of_their_frames(s):
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Shutter(p, "mixed", s)
        view = sc.views[0]
        got = _target(view, "f32", False)
        _ok(p, sc.shutter(got, "f32", PREMUL))
        frames = []
        for i in range(s):
            f = _target(view, "f32", False)
            _ok(p, sc.ex(i, f, "f32", PREMUL))
            frames.append(f)
        # (the samples do differ, in every pixel group the camera and the objects sweep over)
        assert any(frames[i].tobytes() != frames[0].tobytes() for i in range(1, s))
        c = SH.mean([f[..., :3] for f in frames])
        assert got[..., :3].tobytes() == c.tobytes()
        t = SH.mean([(np.float32(1) - f[..., 3]).astype(np.float32) for f in frames])
        assert np.abs(got[..., 3].astype(np.float64) - (1.0 - t.astype(np.float64))).max() <= 2.0 ** -22
        for fmt in ("f16", "u8"):
            for flags, mode in ((0, "opaque"), (PREMUL, "premultiplied")):
                out = _target(view, fmt, False)
                _ok(p, sc.shutter(out, fmt, flags))
                want = O.write_pixel(c, t, mode, OUT_NAME[fmt])
                if fmt == "f16":
                    assert out[..., :3].tobytes() == want[..., :3].tobytes()
                    assert np.abs(out[..., 3].astype(np.float64) - want[..., 3].astype(np.float64)).max() <= 2.0 ** -10
                else:
                    diff = np.abs(out.astype(np.int32) - want.astype(np.int32))
                    assert diff.max() <= 1
                    assert not np.any((diff[..., :3] != 0) & ~O.in_band(c)), mode
    finally:
        p.destroy()


# ---- 4. hooks and launches

@pytest.mark.parametrize("mix", ["quad", "mixed_box"])
def test_hooks_restricted_to_a_sample_are_its_own(mix):
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Shutter(p, mix, 3)
        depths = [_depth(v, 20 + i) for i, v in enumerate(sc.views)]
        _ok(p, sc.shutter(_target(sc.views[0], "f32", False), "f32", 0, depths))
        got = _hooks(p, True)
        wants = []
        for i, v in enumerate(sc.views):
            _ok(p, sc.ex(i, _target(v, "f32", False), "f32", abi.BGS_FLAG_NO_CHUNKS, depths[i]))
            wants.append(_hooks(p, True))
        VS.check_restricted(got, wants, sc.views)
    finally:
        p.destroy()


def test_launch_count_is_the_views_frames_plus_one():
    p = B.GaussianSplattingPlugin(0)
    try:
        for s in (2, 16):
            sc = Shutter(p, "surfel", s)
            _ok(p, sc.views_frame())
            views_count = p.last_launch_count
            _ok(p, sc.shutter(_target(sc.views[0], "f32", False), "f32"))
            assert p.last_launch_count == views_count + 1, (s, views_count, p.last_launch_count)
    finally:
        p.destroy()


# ---- 5. against the oracle

def test_performer_in_the_room_matches_the_mean_of_oracle_frames():
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Shutter(p, "mixed", 4)
        img = _target(sc.views[0], "f32", False)
        _ok(p, sc.shutter(img, "f32"))
        want = np.zeros(img.shape, np.float64)
        for i, v in enumerate(sc.views):
            sts = [st for _, _, _, st in sc.samples[i]]
            want += EO.frame(sc.oracle(i), v.to_abi(), [st.to_abi() for st in sts], [st.num_classes for st in sts],
                             entity_flags=sc.bits)["image"]
        want /= sc.s
        assert float(np.abs(img - want).max()) <= PIXEL_TOL
        assert img[..., :3].any()
    finally:
        p.destroy()


# ---- 6. queued frames, the plugin and the pair-list overflow

def test_queued_frames_and_the_plugin():
    p = B.GaussianSplattingPlugin(0)
    try:
        a, b = Shutter(p, "mixed_conic", 3), Shutter(p, "mixed_conic", 5)
        want = []
        for sc in (a, b):
            out = _target(sc.views[0], "u8", False)
            _ok(p, sc.shutter(out, "u8"))
            want.append(out)
        queued = []
        for sc in (a, b):
            out = _target(sc.views[0], "u8", False)
            _ok(p, sc.shutter(out, "u8", ASYNC))
            queued.append(out)
        assert p.sync()
        for w, q in zip(want, queued):
            assert w.tobytes() == q.tobytes()
        for sc, w in zip((a, b), want):
            got = p.render_shutter(sc.plugin_samples(), sc.views, fmt="rgba8_srgb")
            assert got.shape == w.shape and got.tobytes() == w.tobytes()
        # one depth buffer for every sample, or one per sample
        d = _depth(a.views[0], 7)
        one = p.render_shutter(a.plugin_samples(), a.views, fmt="rgba32f", scene_depths=d, premultiplied=True)
        each = p.render_shutter(a.plugin_samples(), a.views, fmt="rgba32f", scene_depths=[d] * a.s, premultiplied=True)
        raw = _target(a.views[0], "f32", False)
        _ok(p, a.shutter(raw, "f32", PREMUL, [d] * a.s))
        assert one.tobytes() == each.tobytes() == raw.tobytes()
    finally:
        p.destroy()


def test_pair_list_overflow():
    """A shutter frame that outgrows a fresh context's pair buffer re-renders synchronously to the bytes a second render
    gives, blend-over included (the layer goes over the target once); queued on a fresh context, sync() returns
    BGS_NOT_READY and rendering it again gives the same bytes."""
    vs = [B.perspective_view((x, 1.5, 3.0), (x, 1.5, -1.0), 960, 540) for x in (-0.032, 0.032)]
    fill = _noise(vs[0], "f32", 4)
    for queued in (False, True):
        p = B.GaussianSplattingPlugin(0)
        try:
            sc = Shutter(p, "mixed", 2, moving=False, scale=6.0, views=vs)
            first = _target(vs[0], "f32", True, fill)
            if queued:
                _ok(p, sc.shutter(first, "f32", ASYNC | OVER, device=True))
                assert p._lib.bgs_sync(p._ctx) == abi.BGS_NOT_READY
                assert _host(first).tobytes() == fill.tobytes()   # (the truncated frame wrote nothing)
                _ok(p, sc.shutter(first, "f32", ASYNC | OVER, device=True))
                assert p.sync()
            else:
                _ok(p, sc.shutter(first, "f32", OVER, device=True))
            assert p.frame_stats().n_pairs > max(p.frame_stats().n, 1 << 20), p.frame_stats().n_pairs
            second = _target(vs[0], "f32", True, fill)
            _ok(p, sc.shutter(second, "f32", OVER, device=True))
            assert _host(first).tobytes() == _host(second).tobytes()
        finally:
            p.destroy()


# ---- 7. refusals

def test_refusals_write_nothing_and_keep_the_hooks():
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Shutter(p, "mixed", 3)
        view = sc.views[0]
        _ok(p, sc.shutter(_target(view, "f32", False), "f32"))
        hooks = _hooks(p, False)
        base = [entity_settings(st) for st in sc.sts]

        def ents_with(j, **kw):
            e = [abi.bgs_entity_settings.from_buffer_copy(bytes(x)) for x in base]
            for f, val in kw.items():
                setattr(e[j], f, val)
            return e

        def host():
            return np.full((view.height, view.width, 4), 0.5, np.float32)

        def refused(rc, out, want=abi.BGS_EINVAL):
            assert rc == want, p._lib.bgs_last_error(p._ctx)
            assert np.all(_host(out) == 0.5)
            now = _hooks(p, False)
            assert bytes(now["stats"]) == bytes(hooks["stats"])
            for key in ("sorted", "records", "ranges", "entries"):
                assert now[key].tobytes() == hooks[key].tobytes(), key

        # bgs_render_views' refusals, for some sample
        refused(sc.shutter(out := host(), "f32", ents=ents_with(1, draw_mode=9)), out)
        refused(sc.shutter(out := host(), "f32", abi.BGS_FLAG_SORT_ALL), out)
        refused(sc.shutter(out := host(), "f32", ents=ents_with(2, rasterize_mode=int(M.Depth))), out)
        refused(sc.shutter(out := host(), "f32", ents=ents_with(0, rasterize_mode=int(M.OpticalFlow))), out)
        for bad in (float("nan"), float("inf")):   # a Gaussian4d entity's time in one sample
            unis = [[abi.bgs_cloud_uniform.from_buffer_copy(bytes(u)) for u in smp] for smp in sc.unis]
            unis[2][4].time = bad
            refused(sc.shutter(out := host(), "f32", unis=unis), out)
        # s == 0; s k over the limit; views of different sizes
        refused(sc.shutter(out := host(), "f32", unis=[], views=[]), out)
        many = 11   # 11 samples x 6 entities
        refused(sc.shutter(out := host(), "f32", unis=[sc.unis[0]] * many, views=[view] * many), out)
        odd = sc.views[:2] + [V._around((0.0, 1.5, 3.0), 200, 121)]
        refused(sc.shutter(out := host(), "f32", views=odd), out)
        odd = sc.views[:2] + [V._around((0.0, 1.5, 3.0), 199, 120)]
        refused(sc.shutter(out := host(), "f32", views=odd), out)
        # a NULL target; a misaligned device target
        refused(sc.shutter(out := host(), "f32", target=None), out)
        buf = torch.full((view.height * view.width * 4 + 4,), 0.5, dtype=torch.float32, device="cuda")
        refused(sc.shutter(buf, "f32", device=True, target=buf.data_ptr() + 4), buf)
        # a depth buffer one sample cannot read (pitch below its row)
        clouds, es, bits, k, s = sc.common()
        ds = [_depth(v, 1) for v in sc.views]
        zd = (abi.bgs_scene_depth * 3)(*[abi.bgs_scene_depth(depth=d.data_ptr(), pitch_bytes=4 * v.width) for d, v in zip(ds, sc.views)])
        zd[2].pitch_bytes = 4
        us = (abi.bgs_cloud_uniform * (3 * k))(*[u for smp in sc.unis for u in smp])
        vv = (abi.bgs_view * 3)(*[v.to_abi() for v in sc.views])
        out = host()
        refused(p._lib.bgs_render_shutter(p._ctx, clouds, us, es, bits, k, vv, 3, C.byref(s), zd, out.ctypes.data,
                                          abi.BGS_FORMAT_RGBA32F, 0), out)
        # NULL views -> BGS_NOT_READY
        out = host()
        refused(p._lib.bgs_render_shutter(p._ctx, clouds, us, es, bits, k, None, 3, C.byref(s), None, out.ctypes.data,
                                          abi.BGS_FORMAT_RGBA32F, 0), out, abi.BGS_NOT_READY)
    finally:
        p.destroy()


# ---- 8. the C++ host

def test_cpp_host_matches_python(tmp_path):
    """examples/headless.cpp --shutter (include/bgs.hpp's render_shutter: the cloud in 4 samples, sample i moved by
    0.25 i in x) gives the Python host's frame of the same samples."""
    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
    exe = os.path.join(root, "examples", "headless")
    if not os.path.exists(exe):
        subprocess.run(["make", "-C", os.path.join(root, "examples")], check=True)
    n, w, h, scale, s = 3000, 320, 200, 0.3, 4
    raw, cloud_f = tmp_path / "f.raw", tmp_path / "cloud.bin"
    run = subprocess.run([exe, str(n), str(w), str(h), str(scale), str(tmp_path / "0.ppm"), "--raw", str(raw), "--shutter", str(s),
                          "--dump-cloud", str(cloud_f)], capture_output=True, text=True)
    assert run.returncode == 0, run.stderr
    assert f"shutter: {s} samples" in run.stdout and "rendered=1" in run.stdout
    got = np.fromfile(raw, np.uint8)
    g = np.fromfile(cloud_f, np.uint8)[8:].view(np.float32)
    p = B.GaussianSplattingPlugin(0)
    try:
        hd = p.add_cloud(B.PlanarGaussian3d(g[: n * 4].reshape(n, 4), g[n * 4: n * 52].reshape(n, 48),
                                            g[n * 52: n * 56].reshape(n, 4), g[n * 56: n * 60].reshape(n, 4)))
        view, st = B.headless_view(w, h), B.CloudSettings(global_scale=scale)
        samples = []
        for i in range(s):
            m = np.eye(4, dtype=np.float32)
            m[0, 3] = np.float32(0.25) * np.float32(i)
            samples.append([(hd, st, B.CloudTransform(m))])
        img = None
        for _ in range(3):   # (the C++ host renders three frames: the same hints)
            img = p.render_shutter(samples, [view] * s, fmt="rgba8_srgb")
        assert got.tobytes() == img.tobytes()
        assert img[..., :3].any()
    finally:
        p.destroy()
