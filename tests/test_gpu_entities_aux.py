"""bgs_render_entities_aux on the H100: its three frames are bgs_render_entities_ex's frame as given, with every entity in
Depth and with every entity in Normal, byte for byte, in every blend kernel it reaches (entity_aux_cases says which case
reaches which), with and without a depth buffer, in every format, into host and device targets; one entity without a
depth buffer is bgs_render_aux; the frames match the entity oracle; the output flags, the pair-list overflow and the
refusals behave as include/bgs.h rules."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

import bevy_gaussian_splatting_b200 as B
import entity_aux_cases as EA
import entity_cases as E
import scene4d_cases as S4
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import entity_settings
from entity_oracle import entity_oracle as EO

pytestmark = pytest.mark.gpu

PIXEL_TOL = 1e-3
W, H = 200, 120
VIEW = B.headless_view(W, H)
PREV = B.perspective_view((0.2, 1.4, 5.2), (0.0, 1.5, 4.0), W, H)
M = B.RasterizeMode
FORMATS = {"f32": (np.float32, torch.float32, abi.BGS_FORMAT_RGBA32F, 16), "f16": (np.float16, torch.float16, abi.BGS_FORMAT_RGBA16F, 8),
           "u8": (np.uint8, torch.uint8, abi.BGS_FORMAT_RGBA8_SRGB, 4)}


def _extras():
    ex = abi.bgs_render_extras(num_classes=1)
    ex.previous_clip_from_world[:] = PREV.to_abi().clip_from_world[:]
    ex.delta_time = 1.0 / 60.0
    return ex


def _depth(seed, w=W, h=H):
    # (test_gpu_entities' depth buffers: about half the splats of the room lie behind it somewhere)
    return torch.rand((h, w), generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda") * 0.04


class Scene:
    """One case's clouds on a context: the arguments of its bgs_render_entities_ex / _aux calls."""

    def __init__(self, p, listed, flags, view=VIEW):
        self.p, self.view, self.flags = p, view, flags
        up = {}
        self.handles, self.unis, self.sts, self.oracle = [], [], [], []
        for cloud, layout, tr, st in listed:
            if id(cloud) not in up:
                up[id(cloud)] = p.add_cloud(cloud, f16=layout in ("f16", "cov"), precompute_covariance=layout == "cov")
            h = up[id(cloud)]
            self.handles.append(h)
            self.unis.append(p.cloud_uniform(st, tr, h.aabb))
            self.sts.append(st)
            self.oracle.append(E.oracle_entry(cloud, layout, self.unis[-1], st))

    def args(self, sts=None, frame_flags=0, ents=None):
        k = len(self.handles)
        sts = sts or self.sts
        s = sts[0].to_abi()
        s.flags = (s.flags & ~abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX) | frame_flags
        return ((C.c_void_p * k)(*[h._h.value for h in self.handles]), (abi.bgs_cloud_uniform * k)(*self.unis),
                (abi.bgs_entity_settings * k)(*(ents or [entity_settings(st) for st in sts])), (C.c_uint32 * k)(*self.flags), k,
                C.byref(self.view.to_abi()), C.byref(s))

    def ex(self, out, fmt, sts=None, frame_flags=0, depth=None, device=False):
        a = self.args(sts, frame_flags)
        zd = None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * int(self.view.width))
        return self.p._lib.bgs_render_entities_ex(self.p._ctx, *a, C.byref(_extras()), None if zd is None else C.byref(zd),
                                                  _addr(out), FORMATS[fmt][2], int(device))

    def aux(self, outs, fmt, frame_flags=0, depth=None, device=False, ents=None):
        a = self.args(None, frame_flags, ents)
        zd = None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * int(self.view.width))
        return self.p._lib.bgs_render_entities_aux(self.p._ctx, *a, C.byref(_extras()), None if zd is None else C.byref(zd),
                                                   *[_addr(o) for o in outs], FORMATS[fmt][2], int(device))


def _addr(t):
    if t is None:
        return None
    return t.data_ptr() if isinstance(t, torch.Tensor) else t.ctypes.data


def _target(fmt, device, fill=None):
    npd, tod, _, _ = FORMATS[fmt]
    if device:
        t = torch.empty((H, W, 4), dtype=tod, device="cuda")
        if fill is not None:
            t.copy_(torch.from_numpy(fill))
        return t
    return np.empty((H, W, 4), npd) if fill is None else fill.copy()


def _bytes(t):
    if isinstance(t, torch.Tensor):
        torch.cuda.synchronize()
        return t.cpu().numpy().tobytes()
    return t.tobytes()


def _hooks(p, depth_tested):
    fs = p.frame_stats()
    rec, ids = p.projected()
    got = dict(stats=bytes(fs), sorted=p.sorted_entries().tobytes(), records=rec.tobytes(), ids=ids.tobytes(),
               ranges=p.tile_ranges().tobytes(), entries=p.tile_entries().tobytes())
    if depth_tested:
        got["splat_depths"] = p.splat_depths().tobytes()
    return got


def _ok(p, rc):
    assert rc == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)


@pytest.mark.parametrize("case", list(EA.CASES))
@pytest.mark.parametrize("with_depth", [False, True])
def test_aux_frames_are_three_entities_ex_frames(case, with_depth):
    listed, flags = EA.entities(case)
    assert len(EA.kinds([st for _, _, _, st in listed])) == (1 if EA.CASES[case][2] < 3 else (2 if EA.CASES[case][2] == 3 else 3))
    depth = _depth(3) if with_depth else None
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Scene(p, listed, flags)
        for fmt in FORMATS:
            for device in (False, True):
                outs = [_target(fmt, device) for _ in range(3)]
                _ok(p, sc.aux(outs, fmt, depth=depth, device=device))
                torch.cuda.synchronize()
                got = _hooks(p, with_depth)
                for i, sts in enumerate((sc.sts, EA.with_mode(sc.sts, M.Depth), EA.with_mode(sc.sts, M.Normal))):
                    want = _target(fmt, device)
                    _ok(p, sc.ex(want, fmt, sts, depth=depth, device=device))
                    assert _bytes(outs[i]) == _bytes(want), (fmt, device, ["rgba", "depth", "normal"][i])
                    if i == 0:   # hooks and stats: the rgba frame's call's
                        torch.cuda.synchronize()
                        want_hooks = _hooks(p, with_depth)
                        for key in want_hooks:
                            assert got[key] == want_hooks[key], key
    finally:
        p.destroy()


ONE = {"obb3d": dict(), "aabb3d": dict(aabb=True), "aabb2d": dict(gaussian_mode=B.GaussianMode.Gaussian2d, aabb=True)}


@pytest.mark.parametrize("geom", list(ONE))
@pytest.mark.parametrize("layout", ["f32", "f16"])
def test_one_entity_is_render_aux(geom, layout):
    """k == 1 without a depth buffer: bgs_render_aux byte for byte in all three frames, for each colour source it takes,
    with and without HighlightSelected."""
    cloud, _, _, tr, kw = S4.room()[0 if layout == "f32" else 1]
    p = B.GaussianSplattingPlugin(0)
    try:
        h = p.add_cloud(cloud, f16=layout == "f16")
        for mode in (M.Color, M.Depth, M.Position, M.Normal):
            for dm in (B.DrawMode.All, B.DrawMode.HighlightSelected):
                st = B.CloudSettings(**{**kw, **ONE[geom]}, rasterize_mode=mode, draw_mode=dm)
                u = p.cloud_uniform(st, tr, h.aabb)
                for fmt in ("f32", "u8"):
                    want = [_target(fmt, False) for _ in range(3)]
                    s = st.to_abi()
                    _ok(p, p._lib.bgs_render_aux(p._ctx, h._h, C.byref(VIEW.to_abi()), C.byref(u), C.byref(s),
                                                 *[_addr(o) for o in want], FORMATS[fmt][2], 0))
                    got = [_target(fmt, False) for _ in range(3)]
                    e = entity_settings(st)
                    _ok(p, p._lib.bgs_render_entities_aux(p._ctx, (C.c_void_p * 1)(h._h.value), C.byref(u), C.byref(e), None, 1,
                                                          C.byref(VIEW.to_abi()), C.byref(s), None, None,
                                                          *[_addr(o) for o in got], FORMATS[fmt][2], 0))
                    for i in range(3):
                        assert got[i].tobytes() == want[i].tobytes(), (mode.name, dm.name, fmt, i)
        # the plugin: render_view_aux with a depth buffer is this call with k = 1, without one bgs_render_aux
        st = B.CloudSettings(**{**kw, **ONE[geom]})
        depth = _depth(5)
        a = p.render_view_aux(h, st, VIEW, tr)
        b = p.render_view_aux(h, st, VIEW, tr, scene_depth=depth)
        assert all(x.shape == (H, W, 4) for x in a + b)
        assert any(not np.array_equal(x, y) for x, y in zip(a, b))   # (the depth test hides some splats)
        ents = [(h, st, tr)]
        c = p.render_entities_aux(ents, VIEW, scene_depth=depth)
        assert all(np.array_equal(x, y) for x, y in zip(b, c))
    finally:
        p.destroy()


def test_depth_tested_mixed_overlay_frames_match_the_entity_oracle():
    """Quad-uv, conic and surfel entities, one with its overlay, depth-tested: each frame against the entity oracle's frame
    of its colour sources (the rgba frame's Classification entity drawn in Position here, as the oracle tests of
    bgs_render_entities draw the colour sources they check)."""
    listed, flags = EA.entities("mixed_surfel_box")
    c3, l3, t3, s3 = listed[3]
    listed[3] = (c3, l3, t3, dataclasses.replace(s3, rasterize_mode=M.Position))
    depth = _depth(7)
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Scene(p, listed, flags)
        outs = [_target("f32", False) for _ in range(3)]
        _ok(p, sc.aux(outs, "f32", frame_flags=abi.BGS_FLAG_NO_CHUNKS, depth=depth))
        for img, sts in zip(outs, (sc.sts, EA.with_mode(sc.sts, M.Depth), EA.with_mode(sc.sts, M.Normal))):
            want = EO.frame(sc.oracle, VIEW.to_abi(), [st.to_abi() for st in sts], [st.num_classes for st in sts],
                            scene=depth.cpu().numpy(), entity_flags=flags)
            assert np.array_equal(p.sorted_entries(), want["sorted"])
            assert np.array_equal(p.tile_entries(), want["tile_entries"])
            assert float(np.abs(img - want["image"]).max()) <= PIXEL_TOL
    finally:
        p.destroy()


def _nontrivial(fmt, seed):
    rng = np.random.default_rng(seed)
    if fmt == "u8":
        return rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
    return rng.random((H, W, 4), dtype=np.float32).astype(FORMATS[fmt][0])


@pytest.mark.parametrize("fmt", list(FORMATS))
def test_output_flags(fmt):
    """PREMULTIPLIED_OUT: each frame is its _ex frame with the flag.  BLEND_OVER_TARGET into device targets: each frame
    over what its own target holds.  Into host targets: the rgba frame over the context's last frame, the depth and
    normal frames over the previous aux frame's depth and normal frames."""
    listed, flags = EA.entities("mixed_surfel")
    depth = _depth(9)
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Scene(p, listed, flags)
        subs = (sc.sts, EA.with_mode(sc.sts, M.Depth), EA.with_mode(sc.sts, M.Normal))
        pre = abi.BGS_FLAG_PREMULTIPLIED_OUT
        outs = [_target(fmt, False) for _ in range(3)]
        _ok(p, sc.aux(outs, fmt, frame_flags=pre, depth=depth))
        for o, sts in zip(outs, subs):
            want = _target(fmt, False)
            _ok(p, sc.ex(want, fmt, sts, frame_flags=pre, depth=depth))
            assert o.tobytes() == want.tobytes()
        # blend-over, device targets: all three pre-filled with the same frame
        over = abi.BGS_FLAG_BLEND_OVER_TARGET
        base = _nontrivial(fmt, 1)
        outs = [_target(fmt, True, base) for _ in range(3)]
        _ok(p, sc.aux(outs, fmt, frame_flags=over, depth=depth, device=True))
        for o, sts in zip(outs, subs):
            want = _target(fmt, True, base)
            _ok(p, sc.ex(want, fmt, sts, frame_flags=over, depth=depth, device=True))
            assert _bytes(o) == _bytes(want)
        # blend-over, host targets: a first aux frame, then a second one with the flag over it
        first = [_target(fmt, False) for _ in range(3)]
        _ok(p, sc.aux(first, fmt, depth=depth))
        second = [_target(fmt, False, _nontrivial(fmt, 2)) for _ in range(3)]   # (host contents are not read)
        _ok(p, sc.aux(second, fmt, frame_flags=over))
        for o, f, sts in zip(second, first, subs):
            want = _target(fmt, True, f)
            _ok(p, sc.ex(want, fmt, sts, frame_flags=over, device=True))
            assert o.tobytes() == _bytes(want)
    finally:
        p.destroy()


def test_pair_list_overflow_renders_the_frame():
    """A fresh context's first aux frame whose pair list outgrows the first allocation (max(N, 2^20) pairs: the room's
    splats at 6x their scale cover hundreds of tiles each, as kernel_paths' large-footprint inputs do) returns BGS_OK with
    the frames a second render gives."""
    listed, flags = EA.entities("mixed_surfel_box")
    listed = [(c, l, tr, dataclasses.replace(st, global_scale=6.0)) for c, l, tr, st in listed]
    view = B.headless_view(960, 540)
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Scene(p, listed, flags, view)

        def frame():
            outs = [np.empty((540, 960, 4), np.float32) for _ in range(3)]
            a = sc.args()
            _ok(p, p._lib.bgs_render_entities_aux(p._ctx, *a, C.byref(_extras()), None, *[o.ctypes.data for o in outs],
                                                  abi.BGS_FORMAT_RGBA32F, 0))
            return outs

        first = frame()
        n = sum(len(c) for c, _, _, _ in listed)
        assert p.frame_stats().n_pairs > max(n, 1 << 20), p.frame_stats().n_pairs
        second = frame()
        for a, b in zip(first, second):
            assert a.tobytes() == b.tobytes()
    finally:
        p.destroy()


def test_refusals_write_nothing_and_keep_the_hooks():
    listed, flags = EA.entities("mixed")
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Scene(p, listed, flags)
        ok = [_target("f32", False) for _ in range(3)]
        _ok(p, sc.aux(ok, "f32"))
        hooks = _hooks(p, False)
        base = [entity_settings(st) for st in sc.sts]

        def ents_with(j, **kw):
            e = [abi.bgs_entity_settings.from_buffer_copy(bytes(x)) for x in base]
            for f, v in kw.items():
                setattr(e[j], f, v)
            return e

        def refused(rc, outs):
            assert rc == abi.BGS_EINVAL, p._lib.bgs_last_error(p._ctx)
            torch.cuda.synchronize()
            for o in outs:
                if o is not None:
                    assert _bytes(o) == _bytes(_canary(o))
            assert _hooks(p, False) == hooks

        def host():
            return [np.full((H, W, 4), 0.5, np.float32) for _ in range(3)]

        # bgs_render_entities_ex's refusals
        refused(sc.aux(outs := host(), "f32", ents=ents_with(1, draw_mode=9)), outs)
        refused(sc.aux(outs := host(), "f32", ents=ents_with(2, rasterize_mode=int(M.Classification), num_classes=0)), outs)
        refused(sc.aux(outs := host(), "f32", frame_flags=abi.BGS_FLAG_SORT_ALL), outs)
        bad = sc.args()
        bad[3][0] = 2   # (an unknown entity flag)
        outs = host()
        refused(p._lib.bgs_render_entities_aux(p._ctx, *bad, C.byref(_extras()), None, *[o.ctypes.data for o in outs],
                                               abi.BGS_FORMAT_RGBA32F, 0), outs)
        # a NULL target
        for i in range(3):
            outs = host()
            outs[i] = None
            refused(sc.aux(outs, "f32"), outs)
        # a misaligned device target (each of the three)
        for i in range(3):
            buf = [torch.full((H * W * 4 + 4,), 0.5, dtype=torch.float32, device="cuda") for _ in range(3)]
            ptrs = [b.data_ptr() for b in buf]
            ptrs[i] += 4
            a = sc.args()
            refused(p._lib.bgs_render_entities_aux(p._ctx, *a, C.byref(_extras()), None, *ptrs, abi.BGS_FORMAT_RGBA32F, 1), buf)
        # BGS_FLAG_ASYNC; an entity in Velocity
        refused(sc.aux(outs := host(), "f32", frame_flags=abi.BGS_FLAG_ASYNC), outs)
        refused(sc.aux(outs := host(), "f32", ents=ents_with(0, rasterize_mode=int(M.Velocity))), outs)
        # a Gaussian4d cloud; a precomputed-covariance cloud
        perf = S4.performer(500, 9)
        room_cov = S4.room()[2]
        for cloud, layout, st in ((perf, None, S4.settings_4d(B.CloudSettings(), 0.4)),
                                  (room_cov[0], "cov", B.CloudSettings(**room_cov[4]))):
            one = Scene(p, [(cloud, layout, None, st)], [0])
            refused(one.aux(outs := host(), "f32"), outs)
            assert p.render_entities([(one.handles[0], st, None)], VIEW).shape == (H, W, 4)   # (bgs_render_entities_ex takes it)
            _ok(p, sc.aux(ok, "f32"))
            hooks = _hooks(p, False)
    finally:
        p.destroy()


def _canary(o):
    """What a refused call must have left in a target: the fill it was created with."""
    if isinstance(o, torch.Tensor):
        return torch.full_like(o, 0.5)
    return np.full_like(o, 0.5)
