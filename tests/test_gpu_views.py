"""bgs_render_views on the H100: each view's frame is bgs_render_entities_ex's frame of that view, byte for byte, in every
blend kernel a views frame reaches (views_cases says which mix reaches which), for a stereo pair, views of different
sizes and six cube faces, in every format, into host and device targets, with and without per-view depth buffers; the
hooks of the joint frame restricted to a view are that view's own; the launch count does not grow with the views; queued
frames, the pair-list overflow and the refusals behave as include/bgs.h rules; a stereo frame matches the entity oracle."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

import bevy_gaussian_splatting_b200 as B
import entity_cases as E
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


def _ok(p, rc):
    assert rc == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)


def _depth(view, seed):
    # (about half the room's splats lie behind such a buffer somewhere)
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


def _bytes(t):
    if isinstance(t, torch.Tensor):
        torch.cuda.synchronize()
        return t.cpu().numpy().tobytes()
    return t.tobytes()


class Scene:
    """One mix's clouds on a context: the arguments of its bgs_render_views / bgs_render_entities_ex calls."""

    def __init__(self, p, mix, scale=None):
        self.p = p
        listed, self.bits, self.frame_box = V.entities(mix)
        up = {}
        self.handles, self.unis, self.sts, self.oracle = [], [], [], []
        for cloud, layout, tr, st in listed:
            if scale is not None:
                st = dataclasses.replace(st, global_scale=scale)
            if id(cloud) not in up:
                up[id(cloud)] = p.add_cloud(cloud, f16=layout in ("f16", "cov"), precompute_covariance=layout == "cov")
            h = up[id(cloud)]
            self.handles.append(h)
            self.unis.append(p.cloud_uniform(st, tr, h.aabb))
            self.sts.append(st)
            self.oracle.append(E.oracle_entry(cloud, layout, self.unis[-1], st))

    def common(self, flags=0, ents=None):
        k = len(self.handles)
        s = self.sts[0].to_abi()
        s.flags = (s.flags & ~abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX) | flags | (abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX if self.frame_box else 0)
        return ((C.c_void_p * k)(*[h._h.value for h in self.handles]), (abi.bgs_cloud_uniform * k)(*self.unis),
                (abi.bgs_entity_settings * k)(*(ents or [entity_settings(st) for st in self.sts])),
                (C.c_uint32 * k)(*self.bits), k, s)

    def views(self, views, outs, fmt, flags=0, depths=None, device=False, ents=None, targets=None):
        clouds, unis, es, bits, k, s = self.common(flags, ents)
        n = len(views)
        vs = (abi.bgs_view * n)(*[v.to_abi() for v in views])
        zds = None if depths is None else (abi.bgs_scene_depth * n)(
            *[abi.bgs_scene_depth(depth=d.data_ptr(), pitch_bytes=4 * v.width) for d, v in zip(depths, views)])
        tg = targets if targets is not None else (C.c_void_p * n)(*[_addr(o) for o in outs])
        return self.p._lib.bgs_render_views(self.p._ctx, clouds, unis, es, bits, k, vs, n, C.byref(s), zds, tg, FORMATS[fmt][2],
                                            int(device))

    def ex(self, view, out, fmt, flags=0, depth=None, device=False):
        clouds, unis, es, bits, k, s = self.common(flags)
        zd = None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * view.width)
        return self.p._lib.bgs_render_entities_ex(self.p._ctx, clouds, unis, es, bits, k, C.byref(view.to_abi()), C.byref(s),
                                                  None, None if zd is None else C.byref(zd), _addr(out), FORMATS[fmt][2],
                                                  int(device))


def _hooks(p, depth_tested):
    fs = p.frame_stats()
    rec, ids = p.projected()
    got = dict(stats=fs, sorted=p.sorted_entries(), records=rec, ids=ids, ranges=p.tile_ranges(), entries=p.tile_entries())
    got["splat_depths"] = p.splat_depths() if depth_tested else None
    return got


@pytest.mark.parametrize("mix", list(V.MIXES))
@pytest.mark.parametrize("views", V.VIEW_SETS)
@pytest.mark.parametrize("with_depth", [False, True])
def test_each_view_is_its_entities_ex_frame(mix, views, with_depth):
    """Every view's bytes against bgs_render_entities_ex of that view on the same context: all three formats, host and
    device targets, premultiplied output, and blend-over into device targets pre-filled with distinct noise."""
    vs = V.view_set(views)
    depths = [_depth(v, 3 + i) for i, v in enumerate(vs)] if with_depth else None
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Scene(p, mix)
        runs = [(fmt, device, 0) for fmt in FORMATS for device in (False, True)]
        runs += [("f16", False, abi.BGS_FLAG_PREMULTIPLIED_OUT), ("u8", True, abi.BGS_FLAG_PREMULTIPLIED_OUT)]
        for fmt, device, flags in runs:
            outs = [_target(v, fmt, device) for v in vs]
            _ok(p, sc.views(vs, outs, fmt, flags, depths, device))
            for i, v in enumerate(vs):
                want = _target(v, fmt, device)
                _ok(p, sc.ex(v, want, fmt, flags, None if depths is None else depths[i], device))
                assert _bytes(outs[i]) == _bytes(want), (fmt, device, flags, i)
        for fmt in FORMATS:   # blend-over: each device target over its own pixels
            over = abi.BGS_FLAG_BLEND_OVER_TARGET
            noise = [_noise(v, fmt, 10 + i) for i, v in enumerate(vs)]
            outs = [_target(v, fmt, True, f) for v, f in zip(vs, noise)]
            _ok(p, sc.views(vs, outs, fmt, over, depths, True))
            for i, v in enumerate(vs):
                want = _target(v, fmt, True, noise[i])
                _ok(p, sc.ex(v, want, fmt, over, None if depths is None else depths[i], True))
                assert _bytes(outs[i]) == _bytes(want), (fmt, "blend-over", i)
    finally:
        p.destroy()


@pytest.mark.parametrize("mix", ["quad", "mixed_box"])
@pytest.mark.parametrize("views", ["sizes", "cube"])
def test_hooks_restricted_to_a_view_are_its_own(mix, views):
    """View i's entries are the global indices [i n, (i + 1) n): that subsequence of the sorted entries, records, splat
    depths and tile lists is the one-round single-view frame's, and its block of tile ranges gives the same counts."""
    vs = V.view_set(views)
    depths = [_depth(v, 20 + i) for i, v in enumerate(vs)]
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Scene(p, mix)
        _ok(p, sc.views(vs, [_target(v, "f32", False) for v in vs], "f32", 0, depths))
        got = _hooks(p, True)
        wants = []
        for i, v in enumerate(vs):
            _ok(p, sc.ex(v, _target(v, "f32", False), "f32", abi.BGS_FLAG_NO_CHUNKS, depths[i]))
            wants.append(_hooks(p, True))
        VS.check_restricted(got, wants, vs)
    finally:
        p.destroy()


def test_launch_count_does_not_grow_with_the_views_and_one_view_is_entities_ex():
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Scene(p, "mixed")
        stereo, cube = V.view_set("stereo"), V.view_set("cube")
        counts = {}
        for name, vs in (("stereo", stereo), ("cube", cube)):
            _ok(p, sc.views(vs, [_target(v, "f32", False) for v in vs], "f32"))
            counts[name] = p.last_launch_count
        _ok(p, sc.ex(stereo[0], _target(stereo[0], "f32", False), "f32"))
        ex_count = p.last_launch_count
        assert counts["stereo"] == counts["cube"] <= ex_count + 1, (counts, ex_count)
        # v == 1: pixels, hooks, stats and launch count of bgs_render_entities_ex
        for fmt in FORMATS:
            one = [_target(stereo[0], fmt, False)]
            _ok(p, sc.views(stereo[:1], one, fmt))
            got, gl = _hooks(p, False), p.last_launch_count
            want = _target(stereo[0], fmt, False)
            _ok(p, sc.ex(stereo[0], want, fmt))
            ref, rl = _hooks(p, False), p.last_launch_count
            assert one[0].tobytes() == want.tobytes() and gl == rl
            assert bytes(got["stats"]) == bytes(ref["stats"])
            for key in ("sorted", "records", "ids", "ranges", "entries"):
                assert got[key].tobytes() == ref[key].tobytes(), key
    finally:
        p.destroy()


def test_queued_frames_and_the_plugin():
    """Two queued views frames (host targets), then sync(), give the synchronous frames; the plugin's render_views is the
    same call."""
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Scene(p, "mixed_conic")
        a, b = V.view_set("stereo"), V.view_set("sizes")
        want = []
        for vs in (a, b):
            outs = [_target(v, "u8", False) for v in vs]
            _ok(p, sc.views(vs, outs, "u8"))
            want.append(outs)
        queued = []
        for vs in (a, b):
            outs = [_target(v, "u8", False) for v in vs]
            _ok(p, sc.views(vs, outs, "u8", abi.BGS_FLAG_ASYNC))
            queued.append(outs)
        assert p.sync()
        for w, q in zip(want, queued):
            for x, y in zip(w, q):
                assert x.tobytes() == y.tobytes()
        ents = [(h, st, None) for h, st in zip(sc.handles, sc.sts)]
        # (the plugin's uniforms come from the entities' transforms: compare against its own render_entities frames)
        got = p.render_views(ents, b, fmt="rgba8_srgb")
        for v, g in zip(b, got):
            assert g.shape == (v.height, v.width, 4)
            assert g.tobytes() == p.render_entities(ents, v, fmt="rgba8_srgb").tobytes()
    finally:
        p.destroy()


def test_pair_list_overflow():
    """A views frame that outgrows a fresh context's pair buffer re-renders synchronously to the bytes a second render
    gives; queued on a fresh context, sync() returns BGS_NOT_READY and rendering it again gives the same bytes."""
    vs = [B.perspective_view((x, 1.5, 3.0), (x, 1.5, -1.0), 960, 540) for x in (-0.032, 0.032)]
    for queued in (False, True):
        p = B.GaussianSplattingPlugin(0)
        try:
            sc = Scene(p, "mixed", scale=6.0)
            first = [_target(v, "f32", False) for v in vs]
            if queued:
                _ok(p, sc.views(vs, first, "f32", abi.BGS_FLAG_ASYNC))
                assert p._lib.bgs_sync(p._ctx) == abi.BGS_NOT_READY
                _ok(p, sc.views(vs, first, "f32", abi.BGS_FLAG_ASYNC))
                assert p.sync()
            else:
                _ok(p, sc.views(vs, first, "f32"))
            assert p.frame_stats().n_pairs > max(p.frame_stats().n, 1 << 20), p.frame_stats().n_pairs
            second = [_target(v, "f32", False) for v in vs]
            _ok(p, sc.views(vs, second, "f32"))
            for x, y in zip(first, second):
                assert x.tobytes() == y.tobytes()
        finally:
            p.destroy()


def test_stereo_frame_matches_the_entity_oracle():
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Scene(p, "mixed_box")
        vs = V.view_set("stereo")
        outs = [_target(v, "f32", False) for v in vs]
        _ok(p, sc.views(vs, outs, "f32"))
        for v, img in zip(vs, outs):
            want = EO.frame(sc.oracle, v.to_abi(), [st.to_abi() for st in sc.sts], [st.num_classes for st in sc.sts],
                            entity_flags=sc.bits)
            assert float(np.abs(img - want["image"]).max()) <= PIXEL_TOL
    finally:
        p.destroy()


def test_refusals_write_nothing_and_keep_the_hooks():
    vs = V.view_set("sizes")
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Scene(p, "mixed_conic")
        _ok(p, sc.views(vs, [_target(v, "f32", False) for v in vs], "f32"))
        hooks = _hooks(p, False)
        base = [entity_settings(st) for st in sc.sts]

        def ents_with(j, **kw):
            e = [abi.bgs_entity_settings.from_buffer_copy(bytes(x)) for x in base]
            for f, val in kw.items():
                setattr(e[j], f, val)
            return e

        def host():
            return [np.full((v.height, v.width, 4), 0.5, np.float32) for v in vs]

        def refused(rc, outs, want=abi.BGS_EINVAL):
            assert rc == want, p._lib.bgs_last_error(p._ctx)
            torch.cuda.synchronize()
            for o in outs:
                if o is not None:
                    assert np.all(np.asarray(o.cpu() if isinstance(o, torch.Tensor) else o) == 0.5)
            now = _hooks(p, False)
            assert bytes(now["stats"]) == bytes(hooks["stats"])
            for key in ("sorted", "records", "ranges", "entries"):
                assert now[key].tobytes() == hooks[key].tobytes(), key

        # bgs_render_entities_ex's refusals, for some view
        refused(sc.views(vs, outs := host(), "f32", ents=ents_with(1, draw_mode=9)), outs)
        refused(sc.views(vs, outs := host(), "f32", abi.BGS_FLAG_SORT_ALL), outs)
        big = vs[:2] + [B.perspective_view((0.0, 1.5, 3.0), (0.0, 1.5, -1.0), 70000, 8)]
        refused(sc.views(big, outs := host(), "f32"), outs)
        # Depth and OpticalFlow entities
        refused(sc.views(vs, outs := host(), "f32", ents=ents_with(2, rasterize_mode=int(M.Depth))), outs)
        refused(sc.views(vs, outs := host(), "f32", ents=ents_with(0, rasterize_mode=int(M.OpticalFlow))), outs)
        # v == 0; v k over the limit
        refused(sc.views([], [], "f32"), [])
        many = vs * 6   # 18 views x 4 entities
        refused(sc.views(many, outs := [np.full((v.height, v.width, 4), 0.5, np.float32) for v in many], "f32"), outs)
        # a NULL target; a misaligned device target
        outs = host()
        tg = (C.c_void_p * 3)(outs[0].ctypes.data, None, outs[2].ctypes.data)
        refused(sc.views(vs, outs, "f32", targets=tg), outs)
        buf = [torch.full((v.height * v.width * 4 + 4,), 0.5, dtype=torch.float32, device="cuda") for v in vs]
        tg = (C.c_void_p * 3)(buf[0].data_ptr(), buf[1].data_ptr() + 4, buf[2].data_ptr())
        refused(sc.views(vs, buf, "f32", device=True, targets=tg), buf)
        # blend-over into host targets
        refused(sc.views(vs, outs := host(), "f32", abi.BGS_FLAG_BLEND_OVER_TARGET), outs)
        # a depth buffer one view cannot read (pitch below its row)
        clouds, unis, es, bits, k, s = sc.common()
        vv = (abi.bgs_view * 3)(*[v.to_abi() for v in vs])
        ds = [_depth(v, 1) for v in vs]
        zd = (abi.bgs_scene_depth * 3)(*[abi.bgs_scene_depth(depth=d.data_ptr(), pitch_bytes=4 * v.width) for d, v in zip(ds, vs)])
        zd[2].pitch_bytes = 4
        outs = host()
        refused(p._lib.bgs_render_views(p._ctx, clouds, unis, es, bits, k, vv, 3, C.byref(s), zd,
                                        (C.c_void_p * 3)(*[o.ctypes.data for o in outs]), abi.BGS_FORMAT_RGBA32F, 0), outs)
        # NULL views -> BGS_NOT_READY
        outs = host()
        refused(p._lib.bgs_render_views(p._ctx, clouds, unis, es, bits, k, None, 3, C.byref(s), None,
                                        (C.c_void_p * 3)(*[o.ctypes.data for o in outs]), abi.BGS_FORMAT_RGBA32F, 0), outs,
                abi.BGS_NOT_READY)
    finally:
        p.destroy()
