"""bgs_render_views_aux on the H100: each view's colour, depth and normal frames are bgs_render_entities_aux's frames of that
view, byte for byte, in every blend kernel a views aux frame reaches (views_aux_cases says which mix reaches which), for
a stereo pair, views of different sizes and six cube faces, in every format, into host and device targets, with and
without per-view depth buffers; Depth colours are over each view's own range, including its edge cases; one view is
bgs_render_entities_aux; the launch count does not grow with the views; blend-over and the refusals behave as
include/bgs.h rules."""
import ctypes as C

import numpy as np
import pytest
import torch

import bevy_gaussian_splatting_b200 as B
import scene4d_cases as S4
import views_aux_cases as VA
import views_cases as V
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import entity_settings

pytestmark = pytest.mark.gpu

M = B.RasterizeMode
FORMATS = {"f32": (np.float32, torch.float32, abi.BGS_FORMAT_RGBA32F), "f16": (np.float16, torch.float16, abi.BGS_FORMAT_RGBA16F),
           "u8": (np.uint8, torch.uint8, abi.BGS_FORMAT_RGBA8_SRGB)}


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


def _trio(view, fmt, device, fills=None):
    return [_target(view, fmt, device, None if fills is None else fills[f]) for f in range(3)]


def _addr(t):
    return t.data_ptr() if isinstance(t, torch.Tensor) else t.ctypes.data


def _bytes(t):
    if isinstance(t, torch.Tensor):
        torch.cuda.synchronize()
        return t.cpu().numpy().tobytes()
    return t.tobytes()


class Scene:
    """One entity list on a context: the arguments of its bgs_render_views_aux / bgs_render_entities_aux calls."""

    def __init__(self, p, listed, bits=None):
        self.p = p
        up = {}
        self.handles, self.unis, self.sts, self.pos = [], [], [], []
        for cloud, layout, tr, st in listed:
            if id(cloud) not in up:
                up[id(cloud)] = (p.add_cloud(cloud, f16=layout in ("f16", "cov"), precompute_covariance=layout == "cov")
                                 if layout is not None else p.add_cloud(cloud))
            h = up[id(cloud)]
            self.handles.append(h)
            self.unis.append(p.cloud_uniform(st, tr, h.aabb))
            self.sts.append(st)
            self.pos.append(np.asarray(cloud.position_visibility[:, :3], np.float64))
        self.bits = list(bits) if bits is not None else [0] * len(listed)

    def common(self, flags=0, ents=None):
        k = len(self.handles)
        s = self.sts[0].to_abi()
        s.flags = (s.flags & ~abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX) | flags
        return ((C.c_void_p * k)(*[h._h.value for h in self.handles]), (abi.bgs_cloud_uniform * k)(*self.unis),
                (abi.bgs_entity_settings * k)(*(ents or [entity_settings(st) for st in self.sts])),
                (C.c_uint32 * k)(*self.bits), k, s)

    def views_aux(self, views, outs, fmt, flags=0, depths=None, device=False, ents=None, targets=None):
        clouds, unis, es, bits, k, s = self.common(flags, ents)
        n = len(views)
        vs = (abi.bgs_view * max(n, 1))(*[v.to_abi() for v in views])
        zds = None if depths is None else (abi.bgs_scene_depth * n)(
            *[abi.bgs_scene_depth(depth=d.data_ptr(), pitch_bytes=4 * v.width) for d, v in zip(depths, views)])
        tg = targets if targets is not None else [(C.c_void_p * n)(*[_addr(o[f]) for o in outs]) for f in range(3)]
        return self.p._lib.bgs_render_views_aux(self.p._ctx, clouds, unis, es, bits, k, vs, n, C.byref(s), zds, *tg,
                                                FORMATS[fmt][2], int(device))

    def aux(self, view, outs, fmt, flags=0, depth=None, device=False):
        clouds, unis, es, bits, k, s = self.common(flags)
        zd = None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * view.width)
        return self.p._lib.bgs_render_entities_aux(self.p._ctx, clouds, unis, es, bits, k, C.byref(view.to_abi()), C.byref(s),
                                                   None, None if zd is None else C.byref(zd), *[_addr(o) for o in outs],
                                                   FORMATS[fmt][2], int(device))

    def depth_range(self, view):
        """The last frame's (one view's) Depth range: the distances of its sorted[n-1] and sorted[1] from view's camera."""
        srt = self.p.sorted_entries()
        offsets = np.cumsum([0] + [len(x) for x in self.pos])

        def dist(g):
            j = int(np.searchsorted(offsets, g, side="right") - 1)
            m = np.asarray(self.unis[j].transform, np.float64).reshape(4, 4).T   # (column-major)
            pw = m @ np.append(self.pos[j][g - offsets[j]], 1.0)
            return float(np.linalg.norm(pw[:3] - np.asarray(view.to_abi().world_position[:3], np.float64)))

        return dist(int(srt[-1, 1])), dist(int(srt[1, 1]))


def _hooks(p, depth_tested):
    fs = p.frame_stats()
    rec, ids = p.projected()
    got = dict(stats=bytes(fs), sorted=p.sorted_entries().tobytes(), records=rec.tobytes(), ids=ids.tobytes(),
               ranges=p.tile_ranges().tobytes(), entries=p.tile_entries().tobytes())
    if depth_tested:
        got["splat_depths"] = p.splat_depths().tobytes()
    return got


def _room(p, case):
    listed, bits = VA.entities(case)
    return Scene(p, listed, bits)


# (format, device, flags) per view set: together every format into host and device targets, and premultiplied output
RUNS = {"stereo": [("f32", False, 0), ("u8", True, 0), ("f16", True, abi.BGS_FLAG_PREMULTIPLIED_OUT)],
        "sizes": [("f16", False, 0), ("f32", True, 0), ("u8", False, abi.BGS_FLAG_PREMULTIPLIED_OUT)],
        "cube": [("u8", False, 0), ("f16", True, 0), ("f32", True, abi.BGS_FLAG_PREMULTIPLIED_OUT)]}


@pytest.mark.parametrize("case", list(VA.CASES))
@pytest.mark.parametrize("with_depth", [False, True])
def test_each_view_is_its_entities_aux_frames(case, with_depth):
    """Every view's three frames against bgs_render_entities_aux of that view on the same context, for each view set.
    Some two views of each set have different Depth ranges, so a frame-wide range would fail here: in every depth frame,
    and in the rgba frame of the mixes with a Depth entity."""
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = _room(p, case)
        for name in V.VIEW_SETS:
            vs = V.view_set(name)
            depths = [_depth(v, 3 + i) for i, v in enumerate(vs)] if with_depth else None
            for fmt, device, flags in RUNS[name]:
                outs = [_trio(v, fmt, device) for v in vs]
                _ok(p, sc.views_aux(vs, outs, fmt, flags, depths, device))
                ranges = set()
                for i, v in enumerate(vs):
                    want = _trio(v, fmt, device)
                    _ok(p, sc.aux(v, want, fmt, flags, None if depths is None else depths[i], device))
                    ranges.add(sc.depth_range(v))
                    for f in range(3):
                        assert _bytes(outs[i][f]) == _bytes(want[f]), (name, fmt, device, flags, i, f)
                assert len(ranges) >= 2, (name, ranges)
    finally:
        p.destroy()


@pytest.mark.parametrize("with_depth", [False, True])
def test_blend_over_device_targets(with_depth):
    """Blend-over: each device target over its own pixels, as the per-view bgs_render_entities_aux blend-over frames."""
    vs = V.view_set("sizes")
    depths = [_depth(v, 30 + i) for i, v in enumerate(vs)] if with_depth else None
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = _room(p, "mixed_surfel_box")
        over = abi.BGS_FLAG_BLEND_OVER_TARGET
        for fmt in FORMATS:
            noise = [[_noise(v, fmt, 10 + 3 * i + f) for f in range(3)] for i, v in enumerate(vs)]
            outs = [_trio(v, fmt, True, nz) for v, nz in zip(vs, noise)]
            _ok(p, sc.views_aux(vs, outs, fmt, over, depths, True))
            for i, v in enumerate(vs):
                want = _trio(v, fmt, True, noise[i])
                _ok(p, sc.aux(v, want, fmt, over, None if depths is None else depths[i], True))
                for f in range(3):
                    assert _bytes(outs[i][f]) == _bytes(want[f]), (fmt, i, f)
    finally:
        p.destroy()


def test_depth_range_edge_cases():
    """Views with 0 visible gaussians, exactly 1, nothing culled, and some culled, in one frame; and an entity list of one
    gaussian (black Depth colours): each view's frames are its bgs_render_entities_aux frames."""
    views = VA.edge_views()
    vs = list(views.values())
    p = B.GaussianSplattingPlugin(0)
    try:
        cloud = VA.edge_cloud()
        n = len(cloud)
        for listed, check_counts in (([(cloud, "f32", None, B.CloudSettings(rasterize_mode=M.Depth))], True),
                                     ([(cloud, "f32", None, B.CloudSettings(rasterize_mode=M.Depth)),
                                       (cloud, "f32", None, B.CloudSettings(aabb=True))], False),
                                     ([(VA.single_cloud(), "f32", None, B.CloudSettings(rasterize_mode=M.Depth))], False)):
            sc = Scene(p, listed)
            for fmt, device in (("f32", False), ("u8", True)):
                outs = [_trio(v, fmt, device) for v in vs]
                _ok(p, sc.views_aux(vs, outs, fmt, 0, None, device))
                for i, (name, v) in enumerate(views.items()):
                    want = _trio(v, fmt, device)
                    _ok(p, sc.aux(v, want, fmt, 0, None, device))
                    if check_counts:
                        n_vis = p.frame_stats().n_visible
                        assert n_vis == {"none": 0, "one": 1, "all": n, "most": n - 1}.get(name, n_vis), (name, n_vis)
                    for f in range(3):
                        assert _bytes(outs[i][f]) == _bytes(want[f]), (len(listed), fmt, name, f)
    finally:
        p.destroy()


def test_one_view_is_entities_aux_and_the_launch_count_does_not_grow():
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = _room(p, "mixed")
        stereo, cube = V.view_set("stereo"), V.view_set("cube")
        counts = {}
        for name, vs in (("stereo", stereo), ("cube", cube)):
            _ok(p, sc.views_aux(vs, [_trio(v, "f32", False) for v in vs], "f32"))
            counts[name] = p.last_launch_count
        _ok(p, sc.aux(stereo[0], _trio(stereo[0], "f32", False), "f32"))
        assert counts["stereo"] == counts["cube"] == p.last_launch_count, (counts, p.last_launch_count)
        # v == 1: frames, hooks, stats and launch count of bgs_render_entities_aux
        depth = _depth(stereo[0], 7)
        for fmt in FORMATS:
            one = [_trio(stereo[0], fmt, False)]
            _ok(p, sc.views_aux(stereo[:1], one, fmt, 0, [depth]))
            got, gl = _hooks(p, True), p.last_launch_count
            want = _trio(stereo[0], fmt, False)
            _ok(p, sc.aux(stereo[0], want, fmt, 0, depth))
            ref, rl = _hooks(p, True), p.last_launch_count
            assert gl == rl and got == ref
            for f in range(3):
                assert one[0][f].tobytes() == want[f].tobytes(), (fmt, f)
    finally:
        p.destroy()


def test_the_plugin():
    """GaussianSplattingPlugin.render_views_aux is the same call: [rgba, depth, normal] per view, each render_entities_aux's."""
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = _room(p, "quad")
        ents = [(h, st, None) for h, st in zip(sc.handles, sc.sts)]
        vs = V.view_set("sizes")
        got = p.render_views_aux(ents, vs, fmt="rgba8_srgb")
        assert len(got) == len(vs)
        for v, trio in zip(vs, got):
            want = p.render_entities_aux(ents, v, fmt="rgba8_srgb")
            for g, w in zip(trio, want):
                assert g.shape == (v.height, v.width, 4) and g.tobytes() == w.tobytes()
    finally:
        p.destroy()


def test_refusals_write_nothing_and_keep_the_hooks():
    vs = V.view_set("sizes")
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = _room(p, "mixed")
        _ok(p, sc.views_aux(vs, [_trio(v, "f32", False) for v in vs], "f32"))
        hooks = _hooks(p, False)
        base = [entity_settings(st) for st in sc.sts]

        def ents_with(j, **kw):
            e = [abi.bgs_entity_settings.from_buffer_copy(bytes(x)) for x in base]
            for f, val in kw.items():
                setattr(e[j], f, val)
            return e

        def host(views=vs):
            return [[np.full((v.height, v.width, 4), 0.5, np.float32) for _ in range(3)] for v in views]

        def refused(rc, outs, want=abi.BGS_EINVAL):
            assert rc == want, p._lib.bgs_last_error(p._ctx)
            torch.cuda.synchronize()
            for trio in outs:
                for o in trio:
                    assert np.all(np.asarray(o.cpu() if isinstance(o, torch.Tensor) else o) == 0.5)
            assert _hooks(p, False) == hooks

        def arrays(outs):
            return [(C.c_void_p * len(outs))(*[_addr(o[f]) for o in outs]) for f in range(3)]

        # bgs_render_entities_aux's refusals, for some view
        refused(sc.views_aux(vs, outs := host(), "f32", ents=ents_with(1, draw_mode=9)), outs)
        refused(sc.views_aux(vs, outs := host(), "f32", abi.BGS_FLAG_SORT_ALL), outs)
        big = vs[:2] + [B.perspective_view((0.0, 1.5, 3.0), (0.0, 1.5, -1.0), 70000, 8)]
        refused(sc.views_aux(big, outs := host(), "f32"), outs)
        refused(sc.views_aux(vs, outs := host(), "f32", abi.BGS_FLAG_ASYNC), outs)
        refused(sc.views_aux(vs, outs := host(), "f32", ents=ents_with(0, rasterize_mode=int(M.Velocity))), outs)
        refused(sc.views_aux(vs, outs := host(), "f32", ents=ents_with(2, rasterize_mode=int(M.OpticalFlow))), outs)
        # v == 0; v k over the limit
        refused(sc.views_aux([], [], "f32", targets=[(C.c_void_p * 1)()] * 3), [])
        many = vs * 6   # 18 views x 4 entities
        refused(sc.views_aux(many, outs := host(many), "f32"), outs)
        # NULL arrays, a NULL entry, a misaligned device target (in each array)
        for f in range(3):
            outs = host()
            tg = arrays(outs)
            tg[f] = None
            refused(sc.views_aux(vs, outs, "f32", targets=tg), outs)
            outs = host()
            tg = arrays(outs)
            tg[f][1] = None
            refused(sc.views_aux(vs, outs, "f32", targets=tg), outs)
            buf = [[torch.full((v.height * v.width * 4 + 4,), 0.5, dtype=torch.float32, device="cuda") for _ in range(3)]
                   for v in vs]
            tg = arrays(buf)
            tg[f][2] = buf[2][f].data_ptr() + 4
            refused(sc.views_aux(vs, buf, "f32", device=True, targets=tg), buf)
        # blend-over into host targets
        refused(sc.views_aux(vs, outs := host(), "f32", abi.BGS_FLAG_BLEND_OVER_TARGET), outs)
        # a depth buffer one view cannot read (pitch below its row)
        ds = [_depth(v, 1) for v in vs]
        clouds, unis, es, bits, k, s = sc.common()
        vv = (abi.bgs_view * 3)(*[v.to_abi() for v in vs])
        zd = (abi.bgs_scene_depth * 3)(*[abi.bgs_scene_depth(depth=d.data_ptr(), pitch_bytes=4 * v.width) for d, v in zip(ds, vs)])
        zd[2].pitch_bytes = 4
        outs = host()
        refused(p._lib.bgs_render_views_aux(p._ctx, clouds, unis, es, bits, k, vv, 3, C.byref(s), zd, *arrays(outs),
                                            abi.BGS_FORMAT_RGBA32F, 0), outs)
        # NULL views -> BGS_NOT_READY
        outs = host()
        refused(p._lib.bgs_render_views_aux(p._ctx, clouds, unis, es, bits, k, None, 3, C.byref(s), None, *arrays(outs),
                                            abi.BGS_FORMAT_RGBA32F, 0), outs, abi.BGS_NOT_READY)
        # Gaussian4d and precomputed-covariance clouds
        room = S4.room()
        for listed in ([(S4.performer(500, 9), None, None, S4.settings_4d(B.CloudSettings(), 0.3))],
                       [(room[2][0], "cov", room[2][3], B.CloudSettings())]):
            other = Scene(p, listed)
            refused(other.views_aux(vs, outs := host(), "f32"), outs)
    finally:
        p.destroy()
