"""bgs_render_entities on the H100: agreeing entities are bgs_render_scene_4d byte for byte; each entity's records are
its single-cloud call's; frames of mixed blend kinds (quad-uv, conic, surfel, 4D) match the entity oracle, with and
without a depth buffer, queued or not; 2DGS with aabb beside a 4D cloud renders; refusals write nothing."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

import bevy_gaussian_splatting_b200 as B
import blend_cases as BC
import entity_cases as E
import project_cases as PC
import scene4d_cases as S4
import scene_cases as SC
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import entity_settings
from entity_oracle import entity_oracle as EO

pytestmark = pytest.mark.gpu

PIXEL_TOL = 1e-3
W, H = 200, 120
VIEW = B.headless_view(W, H)
PREV = B.perspective_view((0.2, 1.4, 5.2), (0.0, 1.5, 4.0), W, H)
M = B.RasterizeMode
CODES = {np.dtype(np.uint8): abi.BGS_FORMAT_RGBA8_SRGB, np.dtype(np.float16): abi.BGS_FORMAT_RGBA16F,
         np.dtype(np.float32): abi.BGS_FORMAT_RGBA32F}
GEO = [0, 1, 2, 3, 4, 5, 6, 7, 11]


def _extras():
    ex = abi.bgs_render_extras(num_classes=5)
    ex.previous_clip_from_world[:] = PREV.to_abi().clip_from_world[:]
    ex.delta_time = 1.0 / 60.0
    return ex


def _zd(depth):
    return None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * W)


def _load(p, case):
    """(handles, uniforms, settings, oracle entries) of a case; the performer is uploaded once and listed twice."""
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


def render_entities(p, handles, unis, sts, flags=0, ex=None, depth=None, out=None, ents=None):
    k = len(handles)
    clouds = (C.c_void_p * k)(*[h._h.value for h in handles])
    ua = (abi.bgs_cloud_uniform * k)(*unis)
    ea = (abi.bgs_entity_settings * k)(*(ents or [entity_settings(st) for st in sts]))
    s = sts[0].to_abi()
    s.flags |= flags
    return p._lib.bgs_render_entities(p._ctx, clouds, ua, ea, k, C.byref(VIEW.to_abi()), C.byref(s),
                                      None if ex is None else C.byref(ex), None if depth is None else C.byref(_zd(depth)),
                                      out.ctypes.data, CODES[out.dtype], 0)


def render_scene_4d(p, handles, unis, sts, flags=0, ex=None, depth=None, out=None):
    k = len(handles)
    clouds = (C.c_void_p * k)(*[h._h.value for h in handles])
    ua = (abi.bgs_cloud_uniform * k)(*unis)
    wa = (abi.bgs_time_window * k)(*[abi.bgs_time_window(st.time_start, st.time_stop) for st in sts])
    s = sts[0].to_abi()
    s.gaussian_mode = int(sts[0].gaussian_mode if sts[0].gaussian_mode != B.GaussianMode.Gaussian4d else B.GaussianMode.Gaussian3d)
    s.flags |= flags
    return p._lib.bgs_render_scene_4d(p._ctx, clouds, ua, wa, k, C.byref(VIEW.to_abi()), C.byref(s),
                                      None if ex is None else C.byref(ex), None if depth is None else C.byref(_zd(depth)),
                                      out.ctypes.data, CODES[out.dtype], 0)


def capture(p, out, depth_tested):
    torch.cuda.synchronize()
    fs = p.frame_stats()
    got = {"frame": out.tobytes(), "sorted": p.sorted_entries().tobytes(), "stats": bytes(fs), "launches": p.last_launch_count}
    rec, ids = p.projected()
    got["records"], got["ids"] = rec.tobytes(), ids.tobytes()
    if fs.rounds == 1:
        got["ranges"], got["entries"] = p.tile_ranges().tobytes(), p.tile_entries().tobytes()
    if depth_tested:
        got["splat_depths"] = p.splat_depths().tobytes()
    return got


VARIANTS = [(np.float32, 0, False, False), (np.uint8, abi.BGS_FLAG_PREMULTIPLIED_OUT, True, False),
            (np.float16, abi.BGS_FLAG_BLEND_OVER_TARGET, False, True), (np.float32, abi.BGS_FLAG_ASYNC, True, True),
            (np.uint8, abi.BGS_FLAG_CHUNKS, False, False)]


@pytest.mark.parametrize("case", ["agree", "agree_aabb"])
@pytest.mark.parametrize("variant", range(len(VARIANTS)))
def test_agreeing_entities_are_render_scene_4d(case, variant):
    dtype, flags, with_depth, with_ex = VARIANTS[variant]
    depth = torch.rand((H, W), generator=torch.Generator(device="cuda").manual_seed(variant), device="cuda") * 0.04 if with_depth else None
    ex = _extras() if with_ex else None
    got = {}
    for name, fn in (("scene", render_scene_4d), ("entities", render_entities)):
        p = B.GaussianSplattingPlugin(0)   # (a context of its own: blend-over reads the context's last frame)
        try:
            handles, unis, sts, _ = _load(p, case)
            out = np.full((H, W, 4), 0.25 if dtype != np.uint8 else 64, dtype)
            assert fn(p, handles, unis, sts, flags, ex, depth, out) == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)
            if flags & abi.BGS_FLAG_ASYNC:
                assert p.sync()
            got[name] = capture(p, out, depth is not None)
        finally:
            p.destroy()
    for key in got["scene"]:
        assert got["entities"][key] == got["scene"][key], key


def _single(p, h, u, st, ex, depth=None):
    """Records, ids and (under a depth buffer) splat depths of the single-cloud call of one entity (rank order)."""
    s = st.to_abi()
    s.flags |= abi.BGS_FLAG_NO_CHUNKS
    e = abi.bgs_render_extras.from_buffer_copy(bytes(ex))
    e.num_classes = st.num_classes
    out = np.empty((H, W, 4), np.float32)
    if st.gaussian_mode == B.GaussianMode.Gaussian4d:
        rc = p._lib.bgs_render_4d(p._ctx, h._h, C.byref(VIEW.to_abi()), C.byref(u), C.byref(s), C.byref(e),
                                  None if depth is None else C.byref(_zd(depth)), out.ctypes.data, abi.BGS_FORMAT_RGBA32F, 0,
                                  C.c_float(st.time_start), C.c_float(st.time_stop))
    elif depth is not None:
        rc = p._lib.bgs_render_depth_test(p._ctx, h._h, C.byref(VIEW.to_abi()), C.byref(u), C.byref(s), C.byref(e),
                                          C.byref(_zd(depth)), out.ctypes.data, abi.BGS_FORMAT_RGBA32F, 0)
    else:
        rc = p._lib.bgs_render_ex(p._ctx, h._h, C.byref(VIEW.to_abi()), C.byref(u), C.byref(s), C.byref(e), out.ctypes.data,
                                  abi.BGS_FORMAT_RGBA32F, 0)
    assert rc == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)
    rec, ids = p.projected()
    return rec, ids, (p.splat_depths() if depth is not None else None)


@pytest.mark.parametrize("case", ["kinds", "modes", "surfel_4d", "classes"])
@pytest.mark.parametrize("with_depth", [False, True])
def test_records_are_each_entitys_single_cloud_records(case, with_depth):
    """Records, and under a depth buffer splat depths, of every entity (every rasterize mode among the cases) are its
    single-cloud call's bit for bit."""
    p = B.GaussianSplattingPlugin(0)
    try:
        handles, unis, sts, _ = _load(p, case)
        ex = _extras()
        depth = torch.rand((H, W), generator=torch.Generator(device="cuda").manual_seed(11), device="cuda") * 0.04 if with_depth else None
        out = np.empty((H, W, 4), np.float32)
        assert render_entities(p, handles, unis, sts, abi.BGS_FLAG_NO_CHUNKS, ex, depth, out=out) == abi.BGS_OK, \
            p._lib.bgs_last_error(p._ctx)
        rec, ids = p.projected()
        sd = p.splat_depths() if with_depth else None
        sizes = [len(c) for c, _, _, _ in E.entities(case)]
        offs = np.cumsum([0] + sizes)
        for j, (h, u, st) in enumerate(zip(handles, unis, sts)):
            mine = (ids >= offs[j]) & (ids < offs[j + 1])
            local = ids[mine] - offs[j]
            if st.rasterize_mode == M.Velocity and st.gaussian_mode != B.GaussianMode.Gaussian4d:
                assert not S4.drawn(rec[mine]).any() and (rec[mine][:, 8:11] == 0).all()
                continue
            srec, sids, ssd = _single(p, h, u, st, ex, depth)
            pos = np.full(sizes[j], -1)
            pos[sids] = np.arange(len(sids))
            assert (pos[local] >= 0).all(), f"entity {j}: a visible gaussian the single-cloud frame culled"
            want = srec[pos[local]]
            if with_depth:
                assert PC.bits_agree(sd[mine], ssd[pos[local]]).all(), f"entity {j} ({st.rasterize_mode.name}): splat depths"
            # (a Depth colour comes from the joint range, not the cloud's own)
            cols = GEO if st.rasterize_mode == M.Depth else list(range(12))
            assert PC.bits_agree(rec[mine][:, cols], want[:, cols]).all(), f"entity {j} ({st.rasterize_mode.name})"
    finally:
        p.destroy()


@pytest.mark.parametrize("case", ["kinds", "modes", "surfel_4d"])
@pytest.mark.parametrize("with_depth", [False, True])
def test_mixed_kinds_match_the_entity_oracle(case, with_depth):
    p = B.GaussianSplattingPlugin(0)
    try:
        handles, unis, sts, listed = _load(p, case)
        depth = torch.rand((H, W), generator=torch.Generator(device="cuda").manual_seed(7), device="cuda") * 0.04 if with_depth else None
        img = np.empty((H, W, 4), np.float32)
        assert render_entities(p, handles, unis, sts, abi.BGS_FLAG_NO_CHUNKS, depth=depth, out=img) == abi.BGS_OK, \
            p._lib.bgs_last_error(p._ctx)
        want = EO.frame(listed, VIEW.to_abi(), [st.to_abi() for st in sts], [st.num_classes for st in sts],
                        scene=None if depth is None else depth.cpu().numpy())
        assert np.array_equal(p.sorted_entries(), want["sorted"])
        assert p.frame_stats().n_visible == want["n_vis"]
        assert np.array_equal(p.tile_ranges(), want["tile_ranges"])
        assert np.array_equal(p.tile_entries(), want["tile_entries"])
        rec, ids = p.projected()
        assert np.array_equal(ids, want["rank_to_id"])
        # (records: the 4D ones bit for bit, as test_gpu_scene_4d checks them; every record against its single-cloud
        # call in the test above)
        four = ids >= sum(len(c) for c, _, _ in listed[:4])
        assert PC.bits_agree(rec[four][:, GEO], want["records"][four][:, GEO]).all()
        if depth is not None:
            assert PC.bits_agree(p.splat_depths(), want["depths"]).all()
        assert float(np.abs(img - want["image"]).max()) <= PIXEL_TOL
        # queued: the same frame
        q = np.empty((H, W, 4), np.float32)
        assert render_entities(p, handles, unis, sts, abi.BGS_FLAG_NO_CHUNKS | abi.BGS_FLAG_ASYNC, depth=depth, out=q) == abi.BGS_OK
        assert p.sync()
        assert q.tobytes() == img.tobytes()
    finally:
        p.destroy()


def test_refusals_write_nothing():
    p = B.GaussianSplattingPlugin(0)
    try:
        handles, unis, sts, _ = _load(p, "kinds")
        base = [entity_settings(st) for st in sts]

        def with_(j, **kw):
            e = [abi.bgs_entity_settings.from_buffer_copy(bytes(x)) for x in base]
            for f, v in kw.items():
                if f == "window":
                    e[j].window = abi.bgs_time_window(*v)
                else:
                    setattr(e[j], f, v)
            return e

        bad = [with_(0, rasterize_mode=int(M.Classification), num_classes=0),
               with_(0, gaussian_mode=int(B.GaussianMode.Gaussian4d)),
               with_(4, gaussian_mode=int(B.GaussianMode.Gaussian3d)),
               with_(5, rasterize_mode=int(M.Normal)),
               with_(4, window=(0.5, 0.5)),
               with_(5, window=(float("nan"), 1.0)),
               with_(1, draw_mode=9)]
        for ents in bad:
            out = np.full((H, W, 4), 0.5, np.float32)
            assert render_entities(p, handles, unis, sts, out=out, ents=ents) == abi.BGS_EINVAL
            assert (out == 0.5).all()
        out = np.full((H, W, 4), 0.5, np.float32)
        assert render_entities(p, handles, unis, sts, abi.BGS_FLAG_SORT_ALL, out=out) == abi.BGS_EINVAL
        assert (out == 0.5).all()
        # the plugin call: each entity with its own settings, sort bits must agree
        ents = [(h, st, None) for h, st in zip(handles, sts)]
        assert p.render_entities(ents, VIEW).shape == (H, W, 4)
    finally:
        p.destroy()


def _blend_entities(oracle):
    """The blend_cases frames, one entity per blend kind in one 384x256 view: blend_cases' saturated knife-edge frame
    (quad-uv, its knife splats nearest, several at warp corners where the separating-axis cull decides on its slack),
    and saturated conic and surfel frames scattered over the same tiles at depths interleaved with it."""
    knife = BC.knife_case(oracle, "obb3d", True)
    out = [(knife.cloud, knife.settings)]
    for j, geom in enumerate(("aabb3d", "aabb2d")):
        cloud, view, s = BC.saturated_case(geom, n=600, w=384, h=256, seed=3 + j)
        out.append((cloud, s))
    return out, knife.view


@pytest.mark.parametrize("with_depth", [False, True])
def test_mixed_blend_cases_match_the_entity_oracle(oracle, with_depth):
    """Saturated frames: every covered pixel is 0.999 c1 + 0.000999 c2 of its first two covering splats, so a flipped
    coverage decision of any kind moves a pixel by far more than the bound; the GPU frame must stay within 4 ulps of the
    oracle's f32 frame, or 1e-5 where a conic or surfel corner leaves an alpha below the clamp.  Queued equals
    synchronous."""
    ents, view = _blend_entities(oracle)
    w, h = int(view.width), int(view.height)
    p = B.GaussianSplattingPlugin(0)
    try:
        hs = [p.add_cloud(c) for c, _ in ents]
        sts = [s for _, s in ents]
        unis = [p.cloud_uniform(s, None, hh.aabb) for hh, s in zip(hs, sts)]
        depth = None
        if with_depth:
            depth = torch.rand((h, w), generator=torch.Generator(device="cuda").manual_seed(5), device="cuda") * 0.3
        k = len(hs)
        clouds = (C.c_void_p * k)(*[hh._h.value for hh in hs])
        ua = (abi.bgs_cloud_uniform * k)(*unis)
        ea = (abi.bgs_entity_settings * k)(*[entity_settings(s) for s in sts])

        def frame(flags):
            s = sts[0].to_abi()
            s.flags |= flags
            img = np.empty((h, w, 4), np.float32)
            zd = None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * w)
            assert p._lib.bgs_render_entities(p._ctx, clouds, ua, ea, k, C.byref(view.to_abi()), C.byref(s), None,
                                              None if zd is None else C.byref(zd), img.ctypes.data, abi.BGS_FORMAT_RGBA32F,
                                              0) == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)
            if flags & abi.BGS_FLAG_ASYNC:
                assert p.sync()
            return img

        img = frame(0)
        listed = [(c, u, False) for (c, _), u in zip(ents, unis)]
        want = EO.frame(listed, view.to_abi(), [s.to_abi() for s in sts], [1] * k,
                        scene=None if depth is None else depth.cpu().numpy())
        assert np.array_equal(p.sorted_entries(), want["sorted"])
        assert np.array_equal(p.tile_ranges(), want["tile_ranges"])
        assert np.array_equal(p.tile_entries(), want["tile_entries"])
        rec, ids = p.projected()
        assert np.array_equal(ids, want["rank_to_id"])
        offs = np.cumsum([0] + [len(c) for c, _ in ents])
        kind = np.searchsorted(offs, ids, side="right") - 1
        # records of the quad-uv and conic entities bit for bit (the oracle lays a surfel's aabb record out otherwise;
        # the GPU's surfel records are its single-cloud call's, test above, and its coverage shows in the pixels)
        qc = kind < 2
        assert PC.bits_agree(rec[qc][:, GEO], want["records"][qc][:, GEO]).all()
        # each kind is present, and the three share tiles
        r = want["tile_ranges"]
        shared = sum(1 for t in range(len(r)) if r[t, 1] > r[t, 0] and
                     len(set(kind[want["tile_entries"][r[t, 0]:r[t, 1]]].tolist())) == 3)
        assert shared > 0
        wimg = want["image"]
        mag = np.maximum(np.abs(wimg), np.float32(2.0 ** -20)).astype(np.float32)
        bound = np.maximum(4 * np.spacing(mag).astype(np.float64), 1e-5)
        err = np.abs(img.astype(np.float64) - wimg)
        assert (err <= bound).all(), f"{int((err > bound).any(-1).sum())} pixels off, max {err.max()}"
        assert frame(abi.BGS_FLAG_ASYNC).tobytes() == img.tobytes()
    finally:
        p.destroy()


def test_subsets_equal_the_whole():
    """A cloud split into contiguous subsets, each an entity with the settings of the whole (SH degree 2, aabb, Depth),
    renders exactly like the single-cloud call of the whole."""
    st = B.CloudSettings(aabb=True, rasterize_mode=M.Depth, draw_mode=B.DrawMode.HighlightSelected)
    s = st.to_abi()
    s.flags |= abi.BGS_FLAG_NO_CHUNKS
    p = B.GaussianSplattingPlugin(0)
    try:
        cloud = SC.cloud_in_box(4000, 21, sh_degree=2)
        hw = p.add_cloud(cloud)
        u = p.cloud_uniform(st, SC.transform((0.1, 0.0, 0.2)), hw.aabb)
        out = np.zeros((H, W, 4), np.float32)
        assert p._lib.bgs_render_ex(p._ctx, hw._h, C.byref(VIEW.to_abi()), C.byref(u), C.byref(s), None, out.ctypes.data,
                                    abi.BGS_FORMAT_RGBA32F, 0) == abi.BGS_OK
        want = capture(p, out, False)
        parts = [p.subset(hw, ix) for ix in SC.pieces(len(cloud), 3, 21)]
        out = np.zeros((H, W, 4), np.float32)
        assert render_entities(p, parts, [u] * 3, [dataclasses.replace(st, binning_rounds=False)] * 3, out=out) == abi.BGS_OK
        got = capture(p, out, False)
        for key in want:
            assert got[key] == want[key], key
    finally:
        p.destroy()


@pytest.mark.parametrize("i", range(3))
def test_3d_only_agreeing_entities_are_render_scene(i):
    """A 3D-only list (f32 SH degree 2 among the room's layouts) with agreeing settings: bgs_render_scene byte for byte."""
    st = [B.CloudSettings(), B.CloudSettings(aabb=True, rasterize_mode=M.Position),
          B.CloudSettings(gaussian_mode=B.GaussianMode.Gaussian2d, aabb=True, draw_mode=B.DrawMode.Selected)][i]
    depth = torch.rand((H, W), generator=torch.Generator(device="cuda").manual_seed(i), device="cuda") * 0.04 if i != 1 else None
    got = {}
    for name in ("scene", "entities"):
        p = B.GaussianSplattingPlugin(0)
        try:
            handles, unis, sts = [], [], []
            for cloud, layout, _, tr, kw in S4.room()[:2] + [(SC.cloud_in_box(3000, 77, centre=S4.ROOM_CENTRE, sh_degree=2), "f32", 2, None, {})]:
                if i == 2 and layout == "cov":
                    continue
                hh = p.add_cloud(cloud, f16=layout in ("f16", "cov"), precompute_covariance=layout == "cov")
                e = dataclasses.replace(st, **kw)
                handles.append(hh); sts.append(e); unis.append(p.cloud_uniform(e, tr, hh.aabb))
            out = np.zeros((H, W, 4), np.float32)
            if name == "scene":
                k = len(handles)
                s = st.to_abi()
                rc = p._lib.bgs_render_scene(p._ctx, (C.c_void_p * k)(*[x._h.value for x in handles]),
                                             (abi.bgs_cloud_uniform * k)(*unis), k, C.byref(VIEW.to_abi()), C.byref(s), None,
                                             None if depth is None else C.byref(_zd(depth)), out.ctypes.data,
                                             abi.BGS_FORMAT_RGBA32F, 0)
            else:
                rc = render_entities(p, handles, unis, sts, depth=depth, out=out)
            assert rc == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)
            got[name] = capture(p, out, depth is not None)
        finally:
            p.destroy()
    for key in got["scene"]:
        assert got["entities"][key] == got["scene"][key], key
