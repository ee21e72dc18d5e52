"""The projection's and splat depths' grid-stride loops past their first pass, and the scene key-gen's segment walk across
warps, tiles, chunks and CTA ranges, against the CPU oracles (inputs: stride_cases.py; reach: test_oracle_strides.py).

Every frame of A, B and C runs three ways, which must agree byte for byte in every hook, stat and pixel:
* fresh: the first frame of a new context (projection hint n: one pass per warp);
* starved: after a frame of one visible gaussian (hint 1025: a 9-CTA projection grid, a 5-CTA splat-depth grid, so
  every warp strides over groups i, i + 1 and i + 2 of the list: the step the loop's prefetch exists for);
* hinted: the same frame again (hint from the starved frame's visible count).
The starved frame is also checked against the oracle: sorted entries, n_visible, records' geometry, bboxes and
opacities, rank_to_id, tile ranges and entries and splat depths bit for bit; colours within project_cases.colour_bound
(3D) or scene4d_cases.sh_bound (4D); pixels within PIXEL_TOL.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import bevy_gaussian_splatting_b200 as B
import kernel_paths as KP
import project_cases as PC
import scene4d_cases as S4
import scene_cases as SC
import stride_cases as SD
from bevy_gaussian_splatting_b200 import abi
from depth_oracle import depth_oracle as DO
from modes_oracle import modes_oracle as MO
from scene4d_oracle import scene4d_oracle as S4O
from scene_oracle import scene_oracle as SO
from temporal_oracle import temporal_oracle as TO

pytestmark = pytest.mark.gpu

PIXEL_TOL = 1e-3
VIEW = SD.STRIDE_VIEW
W, H = VIEW.width, VIEW.height
RM = B.RasterizeMode
GEO = [0, 1, 2, 3, 4, 5, 6, 7, 11]       # centre, uv rows, bbox, opacity
DT = 1.0 / 60.0


def scene_depth(seed):
    return torch.rand((H, W), generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda") * 0.04


def capture(p, images, depth_tested=False):
    """Everything a frame leaves readable."""
    torch.cuda.synchronize()
    fs = p.frame_stats()
    got = {f"image{i}": np.ascontiguousarray(im).tobytes() for i, im in enumerate(images)}
    got["sorted"], got["stats"] = p.sorted_entries().tobytes(), bytes(fs)
    rec, ids = p.projected()
    got["records"], got["ids"] = rec.tobytes(), ids.tobytes()
    assert fs.rounds == 1
    got["ranges"], got["entries"] = p.tile_ranges().tobytes(), p.tile_entries().tobytes()
    if depth_tested:
        got["splat_depths"] = p.splat_depths().tobytes()
    return got


def starve(p):
    h = p.add_cloud(SD.starve_cloud())
    p.render_view(h, B.CloudSettings(binning_rounds=False), VIEW, to_host=False)
    assert p.frame_stats().n_visible == 1
    h.destroy()


def three_ways(setup, frame):
    """-> (starved capture, setup's state).  setup(p) uploads; frame(p, state) renders and captures.  The starved frame
    runs in a context of its own, alive beside the fresh one, so no value it fails to write can be left over from the
    fresh frame."""
    p, q = B.GaussianSplattingPlugin(0), B.GaussianSplattingPlugin(0)
    try:
        fresh = frame(p, setup(p))
        st = setup(q)
        starve(q)
        starved = frame(q, st)
        hinted = frame(q, st)
        for key in fresh:
            assert starved[key] == fresh[key], f"starved: {key} differs from the fresh frame's"
            assert hinted[key] == fresh[key], f"hinted: {key} differs from the fresh frame's"
        return starved, st
    finally:
        q.destroy()
        p.destroy()


def as_records(cap):
    return np.frombuffer(cap["records"], np.float32).reshape(-1, 12), np.frombuffer(cap["ids"], np.uint32)


def image(cap, i=0):
    return np.frombuffer(cap[f"image{i}"], np.float32).reshape(H, W, 4)


def assert_sorted(cap, sk, si):
    got = np.frombuffer(cap["sorted"], np.uint32).reshape(-1, 2)
    assert np.array_equal(got[:, 0], sk), "sorted keys differ from the oracle's"
    assert np.array_equal(got[:, 1], si), "sort permutation differs from the oracle's"


def assert_tiles(cap, want):
    assert np.frombuffer(cap["stats"][:8], np.uint32)[1] == want["n_vis"]
    assert np.array_equal(np.frombuffer(cap["ranges"], np.uint32).reshape(-1, 2), want["tile_ranges"]), "tile ranges differ"
    assert np.array_equal(np.frombuffer(cap["entries"], np.uint32), want["tile_entries"]), "tile entries differ"
    assert np.array_equal(as_records(cap)[1], want["rank_to_id"]), "rank_to_id differs"


def extras():
    ex = abi.bgs_render_extras(num_classes=SD.NUM_CLASSES)
    ex.previous_clip_from_world[:] = SD.PREV_VIEW.to_abi().clip_from_world[:]
    ex.delta_time = DT
    return ex


# ---------------------------------------------------------------------------------------------------------------------
# A: single 3D clouds at every degree and layout

def single_frame(mode, sort_all, depth):
    s = B.CloudSettings(global_scale=0.8, rasterize_mode=RM.Color if mode is None else mode, num_classes=SD.NUM_CLASSES,
                        sort_all=sort_all, binning_rounds=False)

    def frame(p, st):
        h = st["h"]
        if mode is None:
            return capture(p, p.render_view_aux(h, s, VIEW))
        flow = mode == RM.OpticalFlow
        img = p.render_view(h, s, VIEW, previous_view=SD.PREV_VIEW if flow else None, delta_time=DT if flow else None,
                            scene_depth=depth)
        return capture(p, [img], depth is not None)
    return s, frame


def check_single(oracle, oc, cov, s, mode, cap, u, depth_np=None):
    rec, ids = as_records(cap)
    sk, si = oracle.radix_sort(oracle.keygen(oc.position_visibility, VIEW.to_abi(), u, 32), 32)
    assert_sorted(cap, sk, si)
    base = s.to_abi()
    base.reserved = 1 if cov else 0
    tile_s = abi.bgs_settings.from_buffer_copy(bytes(base))
    if mode in (RM.Classification, RM.OpticalFlow):
        tile_s.rasterize_mode = int(RM.Color)
    til = oracle.render_tiles(oc, VIEW.to_abi(), u, tile_s, want_image=mode not in (RM.Classification, RM.OpticalFlow))
    assert_tiles(cap, til)
    if mode in (RM.Classification, RM.OpticalFlow):
        orec = MO.project_ex(oracle, oc, VIEW.to_abi(), u, base, extras(), ids)
    else:
        orec = oracle.project(oc, VIEW.to_abi(), u, tile_s, ids)
    drawn = orec["xlo"] <= orec["xhi"]
    assert drawn.sum() > 1000
    geo = np.stack([orec[k] for k in ("cx", "cy", "ux", "uy", "vx", "vy")], 1)
    assert PC.bits_agree(rec[drawn, :6], geo[drawn]).all(), "projected geometry not bit-exact"
    bb = rec[:, 6:8].view(np.uint32)
    assert np.array_equal(bb[drawn, 0], orec["xlo"][drawn].astype(np.uint32) | (orec["xhi"][drawn].astype(np.uint32) << 16))
    assert np.array_equal(bb[drawn, 1], orec["ylo"][drawn].astype(np.uint32) | (orec["yhi"][drawn].astype(np.uint32) << 16))
    assert np.all((bb[~drawn, 0] & 0xFFFF) > (bb[~drawn, 0] >> 16)), "a bbox is drawn where the oracle's is empty"
    assert PC.bits_agree(rec[drawn, 11], orec["op"][drawn]).all(), "opacity differs"
    col = np.stack([orec[k] for k in ("r", "g", "b")], 1)[drawn]
    if mode in (RM.Color, None, RM.Classification):
        bound = PC.colour_bound(oc, VIEW, None, int(s.color_space), ids[drawn])
        if mode == RM.Classification:      # mix(sh, hue, 0.5): half the SH colour's error plus one rounding
            bound = bound + np.spacing(np.abs(col).astype(np.float32))
        assert PC.colours_agree(rec[drawn, 8:11], col, bound).all(), "record colour outside its bound"
    elif mode == RM.OpticalFlow:
        assert PC.bits_agree(rec[drawn, 8:11], col).all(), "flow colour differs"
    elif mode != RM.Depth:                 # Normal / Position: the same IEEE operations on both sides
        assert PC.colours_agree(rec[drawn, 8:11], col, np.full(col.shape, 4 * PC.U) * np.maximum(1.0, np.abs(col))).all()
    if depth_np is not None:
        assert PC.bits_agree(np.frombuffer(cap["splat_depths"], np.float32), DO.splat_depth(oc.position_visibility, VIEW.to_abi(), u, ids)).all()
        want = DO.render_tiles(oc, VIEW.to_abi(), u, base, depth_np)
        assert float(np.abs(image(cap) - want).max()) <= PIXEL_TOL
    elif til["image"] is not None:
        assert float(np.abs(image(cap) - til["image"]).max()) <= PIXEL_TOL


@pytest.mark.parametrize("d", [0, 1, 2, 3])
@pytest.mark.parametrize("layout", ["f32", "f16", "cov"])
def test_single_cloud_strides(oracle, layout, d):
    cloud = SD.single_cloud(d, d)
    oc = SC.oracle_cloud(cloud, layout)
    frames = [(name, mode, sort_all, False) for name, mode in SD.single_modes(layout) for sort_all in (False, True)]
    frames.append(("depth_tested", RM.Color, False, True))

    def setup(p):
        h = p.add_cloud(cloud, f16=layout != "f32", precompute_covariance=layout == "cov")
        return dict(h=h)
    for name, mode, sort_all, depth_tested in frames:
        z = scene_depth(d) if depth_tested else None
        s, frame = single_frame(mode, sort_all, z)
        cap, _ = three_ways(setup, frame)
        u = B.GaussianSplattingPlugin.cloud_uniform(s, None, cloud.compute_aabb())
        check_single(oracle, oc, layout == "cov", s, mode, cap, u, None if z is None else z.cpu().numpy())


# ---------------------------------------------------------------------------------------------------------------------
# B: Gaussian4d single clouds

FOUR_D = [(m, sa, False) for m in SD.MODES_4D for sa in (False, True)] + [(RM.Color, False, True), (RM.Velocity, False, True)]


@pytest.mark.parametrize("mode,sort_all,depth_tested", FOUR_D, ids=[f"{m.name}-{'all' if sa else 'compact'}{'-z' if z else ''}"
                                                                      for m, sa, z in FOUR_D])
def test_4d_cloud_strides(oracle, mode, sort_all, depth_tested):
    cloud = SD.performer_4d(0)
    t = SD.STRIDE_4D_TIMES[int(sort_all)]
    s = S4.settings_4d(B.CloudSettings(rasterize_mode=mode, num_classes=SD.NUM_CLASSES, sort_all=sort_all, binning_rounds=False),
                       t, -0.2, 1.1)
    z = scene_depth(11) if depth_tested else None
    flow = mode == RM.OpticalFlow

    def setup(p):
        h = p.add_cloud(cloud)
        u, st, ex = p._call_args(h, s, None, previous_view=SD.PREV_VIEW if flow else None, delta_time=DT if flow else None)
        return dict(h=h, u=u, st=abi.bgs_settings.from_buffer_copy(bytes(st)), ex=ex)

    def frame(p, st):
        img = p.render_view(st["h"], s, VIEW, previous_view=SD.PREV_VIEW if flow else None, delta_time=DT if flow else None,
                            scene_depth=z)
        return capture(p, [img], z is not None)
    cap, st = three_ways(setup, frame)
    ex = st["ex"] if st["ex"] is not None else abi.bgs_render_extras(num_classes=SD.NUM_CLASSES)
    o = TO.frame(cloud, VIEW.to_abi(), st["u"], st["st"], s.time_start, s.time_stop, extras=ex,
                 scene=None if z is None else z.cpu().numpy())
    sk, si = oracle.radix_sort(oracle.keygen(cloud.position_visibility, VIEW.to_abi(), st["u"], 32), 32)
    assert_sorted(cap, sk, si)
    rec, ids = as_records(cap)
    assert np.array_equal(ids, o["rank_to_id"])
    assert PC.bits_agree(rec[:, GEO], o["records"][:, GEO]).all(), "4D record geometry differs"
    drawn = S4.drawn(rec)
    assert 0 < drawn.sum() < 0.8 * len(rec)
    if mode in (RM.Color, RM.Classification):
        bound = S4.sh_bound(cloud, ids[drawn])
        want = o["records"][drawn, 8:11]
        if mode == RM.Classification:
            bound = bound + np.spacing(np.abs(want))
        err = np.abs(rec[drawn, 8:11].astype(np.float64) - want)
        assert (err <= bound).all(), err.max()
    else:
        assert PC.bits_agree(rec[:, 8:11], o["records"][:, 8:11]).all(), "4D record colour differs"
    if z is not None:
        assert PC.bits_agree(np.frombuffer(cap["splat_depths"], np.float32), o["depths"]).all(), "splat depths differ"
    assert float(np.abs(image(cap) - o["image"]).max()) <= PIXEL_TOL


# ---------------------------------------------------------------------------------------------------------------------
# scene calls

def _zd(depth):
    return None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * W)


def render_scene(p, handles, unis, s, windows=None, ex=None, depth=None, out=None, view=VIEW):
    """bgs_render_scene_4d when `windows` is given, else bgs_render_scene, into a host RGBA32F frame."""
    clouds = (C.c_void_p * len(handles))(*[h._h.value for h in handles])
    ua = (abi.bgs_cloud_uniform * len(unis))(*unis)
    a = [C.byref(view.to_abi()), C.byref(s), None if ex is None else C.byref(ex), None if depth is None else C.byref(_zd(depth)),
         out.ctypes.data, abi.BGS_FORMAT_RGBA32F, 0]
    if windows is None:
        return p._lib.bgs_render_scene(p._ctx, clouds, ua, len(handles), *a)
    wa = (abi.bgs_time_window * len(windows))(*[abi.bgs_time_window(*w) for w in windows])
    return p._lib.bgs_render_scene_4d(p._ctx, clouds, ua, wa, len(handles), *a)


# ---------------------------------------------------------------------------------------------------------------------
# C: every projection group in one scene

MIXED = ["color", "classification", "depth", "depth_tested"]


@pytest.mark.parametrize("variant", MIXED)
def test_mixed_scene_strides(variant):
    mode = {"color": RM.Color, "classification": RM.Classification, "depth": RM.Depth, "depth_tested": RM.Color}[variant]
    clouds = SD.mixed_clouds()
    segs = SD.mixed_segments()
    z = scene_depth(21) if variant == "depth_tested" else None
    ex = extras() if mode == RM.Classification else None
    s = B.CloudSettings(rasterize_mode=mode, num_classes=SD.NUM_CLASSES).to_abi()
    s.flags |= abi.BGS_FLAG_NO_CHUNKS

    def cloud_settings(j):
        layout, _, _, _, kw = clouds[j]
        st = B.CloudSettings(rasterize_mode=mode, **kw)
        return S4.settings_4d(st, SD.MIXED_TIME, *SD.MIXED_WINDOW) if layout == "4d" else st

    def setup(p):
        hs = [p.add_cloud(c, f16=layout == "f16") for layout, _, c, _, _ in clouds]
        unis = [p.cloud_uniform(cloud_settings(j), clouds[j][3], hs[j].aabb) for j in range(len(clouds))]
        parts = [p.subset(hs[j], ix.astype(np.uint32)) for j, ix in segs]
        return dict(parts=parts, unis=[unis[j] for j, _ in segs])

    def frame(p, st):
        out = np.empty((H, W, 4), np.float32)
        assert render_scene(p, st["parts"], st["unis"], s, [SD.MIXED_WINDOW] * len(segs), ex, z, out) == abi.BGS_OK, \
            p._lib.bgs_last_error(p._ctx)
        return capture(p, [out], z is not None)
    cap, st = three_ways(setup, frame)
    listed, seg_of, local_of, vis_of = [], [], [], []
    for k, (j, ix) in enumerate(segs):
        layout, _, c, _, _ = clouds[j]
        piece = c.subset(ix)
        listed.append((piece, st["unis"][k], SD.MIXED_WINDOW) if layout == "4d" else (SC.oracle_cloud(piece, layout), st["unis"][k], False))
        seg_of += [j] * len(ix)
        local_of += ix.tolist()
        vis_of += c.position_visibility[ix, 3].tolist()
    seg_of, local_of, vis_of = np.array(seg_of), np.array(local_of), np.array(vis_of, np.float32)
    want = S4O.frame(listed, VIEW.to_abi(), s, extras=ex, scene=None if z is None else z.cpu().numpy())
    if mode == RM.Classification:
        # the scene4d oracle colours 3D records in the four reference modes only: a 3D record's class colour is
        # mix(its Color-frame colour, hue, 0.5) (modes_oracle), and the frame's pixels are held by the three ways alone
        s_col = abi.bgs_settings.from_buffer_copy(bytes(s))
        s_col.rasterize_mode = int(RM.Color)
        col_records = S4O.frame(listed, VIEW.to_abi(), s_col, want_image=False)["records"]
    assert np.array_equal(np.frombuffer(cap["sorted"], np.uint32).reshape(-1, 2), want["sorted"])
    assert_tiles(cap, want)
    rec, ids = as_records(cap)
    assert PC.bits_agree(rec[:, GEO], want["records"][:, GEO]).all(), "scene record geometry differs"
    drawn = S4.drawn(rec)
    for j, (layout, d, c, tr, kw) in enumerate(clouds):
        mine = drawn & (seg_of[ids] == j)
        assert mine.sum() > 50
        got, wc = rec[mine, 8:11], want["records"][mine, 8:11]
        if mode == RM.Depth:
            if layout == "4d":
                assert PC.bits_agree(got, wc).all()
            continue
        if mode == RM.Classification and layout != "4d":
            wc = MO.class_colour(col_records[mine, 8:11], vis_of[ids[mine]], SD.NUM_CLASSES)
        if layout == "4d":
            bound = S4.sh_bound(c, local_of[ids[mine]])
        else:
            bound = PC.colour_bound(SC.oracle_cloud(c, layout), VIEW, tr.matrix, 0, local_of[ids[mine]])
        if mode == RM.Classification:
            bound = bound + np.spacing(np.abs(wc))
        assert PC.colours_agree(got, wc, bound).all(), f"colours of cloud {j} ({layout}, degree {d}) outside their bound"
    if z is not None:
        assert PC.bits_agree(np.frombuffer(cap["splat_depths"], np.float32), want["depths"]).all(), "splat depths differ"
    if mode != RM.Classification:
        assert float(np.abs(image(cap) - want["image"]).max()) <= PIXEL_TOL


# ---------------------------------------------------------------------------------------------------------------------
# D: scene key-gen at scale

def position_planes(pos):
    n = len(pos)
    rot = np.zeros((n, 4), np.float32)
    rot[:, 0] = 1.0
    so = np.empty((n, 4), np.float32)
    so[:, :3], so[:, 3] = 0.01, 0.7
    return rot, so


@pytest.fixture(scope="module")
def keygen_scene():
    sm = KP.device_sm_count()
    if sm != KP.H100_SMS:
        pytest.skip(f"the segment boundaries are placed for {KP.H100_SMS} SMs, this device has {sm}")
    pos = SD.keygen_positions()
    n = len(pos)
    rot, so = position_planes(pos)
    sh48 = np.zeros((n, 48), np.float32)      # (untouched pages: the oracle reads the visible gaussians' only)
    segs = SD.keygen_scene_layout(n, sm)
    p = B.GaussianSplattingPlugin(0)
    h = p.add_cloud(B.PlanarGaussian3d(pos, np.zeros((n, 4), np.float32), rot, so))
    parts = [p.subset(h, np.arange(a, b, dtype=np.uint32)) for a, b in segs]
    host = [B.PlanarGaussian3d(pos[a:b], sh48[a:b], rot[a:b], so[a:b]) for a, b in segs]
    yield dict(p=p, h=h, parts=parts, host=host, segs=segs,
               whole=B.PlanarGaussian3d(pos, sh48, rot, so))
    p.destroy()


def _render(p, handles, unis, s, queued, depth=None):
    out = np.empty((H, W, 4), np.float32)
    s2 = abi.bgs_settings.from_buffer_copy(bytes(s))
    if queued:
        s2.flags |= abi.BGS_FLAG_ASYNC
    assert render_scene(p, handles, unis, s2, depth=depth, out=out) == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)
    if queued:
        assert p.sync()
    return capture(p, [out], depth is not None)


def test_keygen_scene_mixed_uniforms_queued_and_synchronous(keygen_scene):
    ks = keygen_scene
    p = ks["p"]
    trs = SD.keygen_transforms()
    unis = [p.cloud_uniform(B.CloudSettings(global_scale=trs[i][1]), trs[i][0], ks["h"].aabb)
            for i in (SD.keygen_uniform_index(j, a) for j, (a, _) in enumerate(ks["segs"]))]
    s = B.CloudSettings().to_abi()
    s.flags |= abi.BGS_FLAG_NO_CHUNKS
    queued = _render(p, ks["parts"], unis, s, True)
    listed = [(c, u, False) for c, u in zip(ks["host"], unis)]
    want_sorted = SO.sorted_entries(listed, VIEW.to_abi())
    assert np.array_equal(np.frombuffer(queued["sorted"], np.uint32).reshape(-1, 2), want_sorted), \
        "sorted entries (with the culled tail) differ from the scene oracle's"
    want = SO.render_tiles(listed, VIEW.to_abi(), s)
    assert want["n_vis"] > 50_000
    assert_tiles(queued, want)
    assert float(np.abs(image(queued) - want["image"]).max()) <= PIXEL_TOL
    sync = _render(p, ks["parts"], unis, s, False)
    for key in queued:
        assert sync[key] == queued[key], f"synchronous frame: {key} differs from the queued one"


def test_keygen_scene_split_is_the_whole_cloud(keygen_scene):
    """One uniform for every segment: the scene is the whole cloud cut at every boundary of the layout."""
    ks = keygen_scene
    p, h = ks["p"], ks["h"]
    st = B.CloudSettings(global_scale=1.2)
    u = p.cloud_uniform(st, SC.transform((0.02, -0.01, 0.03)), h.aabb)
    s = st.to_abi()
    s.flags |= abi.BGS_FLAG_NO_CHUNKS
    z = scene_depth(31)
    out = np.empty((H, W, 4), np.float32)
    assert p._lib.bgs_render_depth_test(p._ctx, h._h, C.byref(VIEW.to_abi()), C.byref(u), C.byref(s), None, C.byref(_zd(z)),
                                        out.ctypes.data, abi.BGS_FORMAT_RGBA32F, 0) == abi.BGS_OK
    whole = capture(p, [out], True)
    assert np.frombuffer(whole["stats"][:8], np.uint32)[1] > 50_000
    for queued in (True, False):
        got = _render(p, ks["parts"], [u] * len(ks["parts"]), s, queued, z)
        for key in whole:
            assert got[key] == whole[key], f"{'queued' if queued else 'synchronous'} split: {key} differs from the whole cloud's"
