"""bgs_render_entities_many and _pick_many on the H100: at k <= 64 each is its capped call byte for byte (pixels in three
formats and output modes, every hook, stats and launch count, pick records); above 64 a cloud split into k contiguous
subsets renders exactly like the whole (f32, f16 and covariance layouts, SH degrees 0-3, queued and chunked frames, a
Gaussian4d cloud, the pick frame); mixed entity lists of 65 and 300 match the entity oracle; queued frames keep their
tables; a particle step between two frames is seen by the second only; refusals name the entity and keep the hooks."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

import bevy_gaussian_splatting_b200 as B
import entities_many_cases as EM
import entity_cases as E
import project_cases as PC
import scene4d_cases as S4
import scene_cases as SC
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.particles import random_particle_behaviors
from entity_oracle import entity_oracle as EO

pytestmark = pytest.mark.gpu

W, H = 200, 120
VIEW = B.headless_view(W, H)
PREV = B.perspective_view((0.2, 1.4, 5.2), (0.0, 1.5, 4.0), W, H)
M, G = B.RasterizeMode, B.GaussianMode
CODES = {np.dtype(np.uint8): abi.BGS_FORMAT_RGBA8_SRGB, np.dtype(np.float16): abi.BGS_FORMAT_RGBA16F,
         np.dtype(np.float32): abi.BGS_FORMAT_RGBA32F}
PIXEL_TOL = 1e-3
GEO = [0, 1, 2, 3, 4, 5, 6, 7, 11]


def _extras(num_classes=5):
    ex = abi.bgs_render_extras(num_classes=num_classes)
    ex.previous_clip_from_world[:] = PREV.to_abi().clip_from_world[:]
    ex.delta_time = 1.0 / 60.0
    return ex


def _depth(seed, w=W, h=H):
    return torch.rand((h, w), generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda") * 0.04


def _load(p, listed, view=VIEW, flags=None):
    """An entity list [(cloud, layout, transform, CloudSettings)] uploaded into p (each cloud once) as EM.Entities, and its
    oracle entries."""
    up, handles, unis, sts, oracle = {}, [], [], [], []
    for cloud, layout, tr, st in listed:
        if id(cloud) not in up:
            up[id(cloud)] = p.add_cloud(cloud, f16=layout in ("f16", "cov"), precompute_covariance=layout == "cov")
        h = up[id(cloud)]
        handles.append(h)
        unis.append(p.cloud_uniform(st, tr, h.aabb))
        sts.append(st)
        oracle.append(E.oracle_entry(cloud, layout, unis[-1], st))
    return EM.Entities(p, handles, unis, sts, view, flags), oracle


def capture(p, out, depth_tested):
    torch.cuda.synchronize()
    fs = p.frame_stats()
    got = {"frame": out.tobytes() if isinstance(out, np.ndarray) else out.cpu().numpy().tobytes(),
           "sorted": p.sorted_entries().tobytes(), "stats": bytes(fs)}
    rec, ids = p.projected()
    got["records"], got["ids"] = rec.tobytes(), ids.tobytes()
    if fs.rounds == 1:
        got["ranges"], got["entries"] = p.tile_ranges().tobytes(), p.tile_entries().tobytes()
    if depth_tested:
        got["splat_depths"] = p.splat_depths().tobytes()
    return got


def _rendered(p, call, flags):
    """call() until its frame is complete: a queued frame that outgrew the pair buffer (bgs_sync's BGS_NOT_READY, the
    buffer now grown) is rendered again, as the rule of BGS_FLAG_ASYNC asks."""
    for _ in range(3):
        EM.ok(p, call())
        if not flags & abi.BGS_FLAG_ASYNC or p.sync():
            return
    raise AssertionError("the queued frame kept outgrowing the pair buffer")


def _same(got, want):
    assert got.keys() == want.keys()
    for key in want:
        assert got[key] == want[key], key


# ---- 1. identity at k <= 64: bgs_render_entities_many is bgs_render_entities_ex, launch count included

VARIANTS = [(np.float32, 0, False), (np.uint8, abi.BGS_FLAG_PREMULTIPLIED_OUT, True),
            (np.float16, abi.BGS_FLAG_BLEND_OVER_TARGET, False), (np.float32, abi.BGS_FLAG_ASYNC, True),
            (np.uint8, abi.BGS_FLAG_CHUNKS, False), (np.float16, abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX, True)]


@pytest.mark.parametrize("case", list(E.CASES))
def test_many_is_ex_at_k_le_64(case):
    """Every entity_cases case, in every variant in turn on one context per call: the same frames, hooks and launches."""
    got = {}
    for name in ("ex", "many"):
        p = B.GaussianSplattingPlugin(0)
        try:
            ents, _ = _load(p, E.entities(case), flags=[j & 1 for j in range(6)])
            got[name] = []
            for i, (dtype, flags, with_depth) in enumerate(VARIANTS):
                depth = _depth(i) if with_depth else None
                out = np.full((H, W, 4), 0.25 if dtype != np.uint8 else 64, dtype)
                EM.ok(p, ents.call(name, out, CODES[np.dtype(dtype)], flags, depth, _extras()))
                if flags & abi.BGS_FLAG_ASYNC:
                    assert p.sync()
                cap = capture(p, out, depth is not None)
                cap["launches"] = p.last_launch_count
                got[name].append(cap)
        finally:
            p.destroy()
    for g, w in zip(got["many"], got["ex"]):
        _same(g, w)


PICK_VARIANTS = [(np.float32, 0, False, False), (np.uint8, abi.BGS_FLAG_PREMULTIPLIED_OUT, True, True),
                 (np.float16, abi.BGS_FLAG_BLEND_OVER_TARGET, True, False), (np.float32, abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX, False, True)]


@pytest.mark.parametrize("case", list(E.CASES))
def test_pick_many_is_pick_at_k_le_64(case):
    """Every entity_cases case through bgs_render_entities_pick_many and _pick: pixels, pick records (host and device
    targets), hooks, splat depths and launch count."""
    got = {}
    for name in ("pick", "pick_many"):
        p = B.GaussianSplattingPlugin(0)
        try:
            ents, _ = _load(p, E.entities(case), flags=[(j + 1) & 1 for j in range(6)])
            got[name] = []
            for i, (dtype, flags, with_depth, device) in enumerate(PICK_VARIANTS):
                depth = _depth(10 + i) if with_depth else None
                if device:
                    tdt = {np.dtype(np.uint8): torch.uint8, np.dtype(np.float16): torch.float16}.get(np.dtype(dtype), torch.float32)
                    out = torch.zeros((H, W, 4), dtype=tdt, device="cuda")
                    pick = torch.zeros((H, W, 4), dtype=torch.int32, device="cuda")
                else:
                    out = np.full((H, W, 4), 0.25 if dtype != np.uint8 else 64, dtype)
                    pick = np.zeros((H, W), abi.PICK_DTYPE)
                EM.ok(p, ents.call(name, out, CODES[np.dtype(dtype)], flags, depth, _extras(), device=device, pick=pick))
                cap = capture(p, out, True)
                torch.cuda.synchronize()
                cap["pick"] = pick.tobytes() if isinstance(pick, np.ndarray) else pick.cpu().numpy().tobytes()
                cap["launches"] = p.last_launch_count
                got[name].append(cap)
        finally:
            p.destroy()
    for g, w in zip(got["pick_many"], got["pick"]):
        _same(g, w)


# ---- 2. split identity above 64: k contiguous subsets, each an entity with the whole's uniform and settings

SV = B.headless_view(256, 192)
SPLITS = [  # (k, layout, SH degree, settings overrides, frame flags, depth buffer)
    (65, "f32", 3, dict(), 0, True),
    (257, "f16", 1, dict(aabb=True), abi.BGS_FLAG_ASYNC, False),
    (257, "f32", 2, dict(rasterize_mode=M.Depth, draw_mode=B.DrawMode.HighlightSelected), 0, True),
    (4097, "cov", 3, dict(), abi.BGS_FLAG_CHUNKS, False),
    (4097, "f16", 2, dict(gaussian_mode=G.Gaussian2d, aabb=True), abi.BGS_FLAG_ASYNC, True),
    (65536, "f32", 0, dict(), 0, True),
    (65536, "f16", 3, dict(), abi.BGS_FLAG_ASYNC | abi.BGS_FLAG_CHUNKS, False),
]


def _whole_frame(p, h, u, st, flags, depth, out, view=SV):
    s = st.to_abi()
    s.flags |= flags
    v = view.to_abi()
    if depth is not None:
        zd = abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * view.width)
        return p._lib.bgs_render_depth_test(p._ctx, h._h, C.byref(v), C.byref(u), C.byref(s), None, C.byref(zd), out.ctypes.data,
                                            abi.BGS_FORMAT_RGBA32F, 0)
    return p._lib.bgs_render_ex(p._ctx, h._h, C.byref(v), C.byref(u), C.byref(s), None, out.ctypes.data, abi.BGS_FORMAT_RGBA32F, 0)


@pytest.mark.parametrize("i", range(len(SPLITS)))
def test_split_equals_the_whole(i):
    k, layout, d, over, flags, with_depth = SPLITS[i]
    n = max(40 * k, 3 * 8 * EM.KG_TILE + 33 * k)
    st = B.CloudSettings(**over)
    p = B.GaussianSplattingPlugin(0)
    try:
        cloud = SC.cloud_in_box(n, 60 + i, half=1.6, scale=0.03, sh_degree=d)
        hw = p.add_cloud(cloud, f16=layout in ("f16", "cov"), precompute_covariance=layout == "cov")
        u = p.cloud_uniform(st, SC.transform((0.1, 0.0, 0.2), 1.05, 0.3), hw.aabb)
        depth = _depth(20 + i, SV.width, SV.height) if with_depth else None
        frame_flags = flags if flags & abi.BGS_FLAG_CHUNKS else flags | abi.BGS_FLAG_NO_CHUNKS
        want_img = np.zeros((SV.height, SV.width, 4), np.float32)
        _rendered(p, lambda: _whole_frame(p, hw, u, st, frame_flags, depth, want_img), flags)
        want = capture(p, want_img, with_depth)
        parts = [p.subset(hw, ix) for ix in EM.pieces(n, k, i)]
        ents = EM.Entities(p, parts, [u] * k, [st] * k, SV)
        img = np.zeros((SV.height, SV.width, 4), np.float32)
        _rendered(p, lambda: ents.call("many", img, abi.BGS_FORMAT_RGBA32F, frame_flags, depth), flags)
        _same(capture(p, img, with_depth), want)
    finally:
        p.destroy()


@pytest.mark.parametrize("k", [65, 300])
def test_split_4d_equals_render_4d(k):
    """A Gaussian4d cloud split into k subsets, each entity in the whole's window, is bgs_render_4d of the whole."""
    n = 40 * k
    st = S4.settings_4d(B.CloudSettings(global_opacity=0.9), 0.45, -0.2, 1.1)
    p = B.GaussianSplattingPlugin(0)
    try:
        cloud = S4.performer(n, 77, centre=(0.0, 1.5, -1.0), spread=1.4, scale=0.05)
        hw = p.add_cloud(cloud)
        u = p.cloud_uniform(st, SC.transform((0.0, 0.1, 0.0), 1.0, 0.2), hw.aabb)
        depth = _depth(30 + k, SV.width, SV.height)
        zd = abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * SV.width)
        s = st.to_abi()
        s.flags |= abi.BGS_FLAG_NO_CHUNKS
        want_img = np.zeros((SV.height, SV.width, 4), np.float32)
        EM.ok(p, p._lib.bgs_render_4d(p._ctx, hw._h, C.byref(SV.to_abi()), C.byref(u), C.byref(s), None, C.byref(zd),
                                      want_img.ctypes.data, abi.BGS_FORMAT_RGBA32F, 0, C.c_float(st.time_start),
                                      C.c_float(st.time_stop)))
        want = capture(p, want_img, True)
        parts = [p.subset(hw, ix) for ix in EM.pieces(n, k, 5)]
        ents = EM.Entities(p, parts, [u] * k, [st] * k, SV)
        img = np.zeros((SV.height, SV.width, 4), np.float32)
        EM.ok(p, ents.call("many", img, abi.BGS_FORMAT_RGBA32F, abi.BGS_FLAG_NO_CHUNKS, depth))
        _same(capture(p, img, True), want)
    finally:
        p.destroy()


def test_split_pick_maps_to_the_whole():
    """The pick frame of a cloud split into 4097 subsets: entity j, index i is (0, o_j + i) of the whole's one-entity pick
    frame, with its weight and depth bit for bit; the colour frames are byte-equal."""
    k, n = 4097, 4097 * 40
    st = B.CloudSettings(aabb=True)
    p = B.GaussianSplattingPlugin(0)
    try:
        cloud = SC.cloud_in_box(n, 91, half=1.6, scale=0.03, sh_degree=1)
        hw = p.add_cloud(cloud)
        u = p.cloud_uniform(st, None, hw.aabb)
        depth = _depth(41, SV.width, SV.height)
        one = EM.Entities(p, [hw], [u], [st], SV)
        want_img = np.zeros((SV.height, SV.width, 4), np.float32)
        want = np.zeros((SV.height, SV.width), abi.PICK_DTYPE)
        EM.ok(p, one.call("pick", want_img, abi.BGS_FORMAT_RGBA32F, 0, depth, pick=want))
        cuts = np.array(EM.split_cuts(n, k, 2), np.int64)
        parts = [p.subset(hw, np.arange(a, b)) for a, b in zip(cuts[:-1], cuts[1:])]
        ents = EM.Entities(p, parts, [u] * k, [st] * k, SV)
        img = np.zeros((SV.height, SV.width, 4), np.float32)
        got = np.zeros((SV.height, SV.width), abi.PICK_DTYPE)
        EM.ok(p, ents.call("pick_many", img, abi.BGS_FORMAT_RGBA32F, 0, depth, pick=got))
        assert img.tobytes() == want_img.tobytes()
        hit = got["entity"] != abi.BGS_PICK_NONE
        assert np.array_equal(hit, want["entity"] != abi.BGS_PICK_NONE) and hit.sum() > 1000
        assert got["entity"][hit].max() > 63
        glob = cuts[got["entity"][hit].astype(np.int64)] + got["index"][hit]
        assert np.array_equal(glob, want["index"][hit].astype(np.int64)) and (want["entity"][hit] == 0).all()
        assert got["weight"].tobytes() == want["weight"].tobytes() and got["depth"].tobytes() == want["depth"].tobytes()
    finally:
        p.destroy()


# ---- 3. the entity oracle above 64 entities

def _oracle_list(k, seed=0):
    """k entities: the room's clouds and the 4D performer (at staggered times) under their own transforms with mixed draw
    modes, colour sources (Classification and OpticalFlow on the performer), overlays, 2DGS surfels and conics, and
    (k > 200) one small cloud listed 200 times on a grid."""
    rng = np.random.default_rng(seed)
    base = E.entities("kinds")
    modes = [dict(), dict(aabb=True), dict(gaussian_mode=G.Gaussian2d, aabb=True), dict(rasterize_mode=M.Classification, num_classes=3),
             dict(rasterize_mode=M.OpticalFlow), dict(draw_mode=B.DrawMode.HighlightSelected), dict(rasterize_mode=M.Position)]
    modes_3d = [m for m in modes if m.get("rasterize_mode") not in (M.Classification, M.OpticalFlow)]
    small = SC.cloud_in_box(120, 300 + seed, centre=(0.0, 0.0, 0.0), half=0.15, scale=0.05, sh_degree=2)
    out = []
    for j in range(k):
        if k > 200 and j >= k - 200:
            g = j - (k - 200)
            tr = SC.transform(((g % 20) * 0.18 - 1.7, 1.5 + (g // 20) * 0.16 - 0.8, -2.5 - 0.02 * (g % 7)), 1.0, 0.1 * g)
            out.append((small, "f32", tr, B.CloudSettings(**modes[g % 3])))
            continue
        cloud, layout, _, st = base[j % 6]
        tr = SC.transform(tuple(rng.uniform(-0.8, 0.8, 3) * (1.0, 0.5, 0.6)), float(rng.uniform(0.6, 1.1)), float(rng.uniform(-1, 1)))
        if layout is None:   # the performer, at its own time
            t = 0.1 + 0.8 * (j % 9) / 8.0
            over = modes[j % 7] if modes[j % 7].get("gaussian_mode") is None else dict(aabb=True)
            st = S4.settings_4d(dataclasses.replace(B.CloudSettings(global_opacity=0.9), **over), t, -0.2, 1.1)
        elif layout == "cov":   # (no rotation: Gaussian3d, and no Normal)
            st = B.CloudSettings(**[dict(), dict(aabb=True), dict(rasterize_mode=M.Position)][j % 3])
        else:   # (the oracle draws Classification and OpticalFlow on Gaussian4d entities only)
            st = B.CloudSettings(**modes_3d[j % len(modes_3d)])
        out.append((cloud, layout, tr, st))
    return out


@pytest.mark.parametrize("k,with_depth", [(65, False), (300, True)])
def test_many_matches_the_entity_oracle(k, with_depth):
    p = B.GaussianSplattingPlugin(0)
    try:
        listed = _oracle_list(k, k)
        ents, oracle = _load(p, listed, flags=[1 if j % 11 == 3 else 0 for j in range(k)])
        depth = _depth(50 + k) if with_depth else None
        img = np.empty((H, W, 4), np.float32)
        ex = _extras()
        EM.ok(p, ents.call("many", img, abi.BGS_FORMAT_RGBA32F, abi.BGS_FLAG_NO_CHUNKS, depth, ex))
        want = EO.frame(oracle, VIEW.to_abi(), [st.to_abi() for st in ents.sts], [st.num_classes for st in ents.sts], extras=ex,
                        scene=None if depth is None else depth.cpu().numpy(), entity_flags=list(ents.flags))
        assert np.array_equal(p.sorted_entries(), want["sorted"])
        assert p.frame_stats().n_visible == want["n_vis"]
        assert np.array_equal(p.tile_ranges(), want["tile_ranges"])
        assert np.array_equal(p.tile_entries(), want["tile_entries"])
        rec, ids = p.projected()
        assert np.array_equal(ids, want["rank_to_id"])
        # (records: the 4D ones bit for bit, as test_gpu_entities checks them)
        offsets = np.cumsum([0] + [len(c) for c, _, _ in oracle])
        four = np.array([listed[j][1] is None for j in range(k)])[np.searchsorted(offsets, ids, side="right") - 1]
        assert four.any()
        assert PC.bits_agree(rec[four][:, GEO], want["records"][four][:, GEO]).all()
        if depth is not None:
            assert PC.bits_agree(p.splat_depths(), want["depths"]).all()
        assert float(np.abs(img - want["image"]).max()) <= PIXEL_TOL
    finally:
        p.destroy()


def test_khr_scene_with_many_placements(tmp_path):
    """A KHR_gaussian_splatting scene whose one mesh is placed by 90 nodes loads as 90 bundles of one primitive, becomes
    one resident cloud listed 90 times through add_scene, and renders through render_entities_many as the entity oracle
    does."""
    import base64
    import json

    from bevy_gaussian_splatting_b200.khr import SceneExportCloud, encode_scene, load_scene

    cloud = SC.cloud_in_box(150, 7, centre=(0.0, 0.0, 0.0), half=0.2, scale=0.06, sh_degree=1)
    root, binary = encode_scene([SceneExportCloud(cloud, "c")])
    (node,) = root["nodes"]
    root["nodes"] = []
    for j in range(90):
        m = SC.transform(((j % 10) * 0.3 - 1.4, 1.5 + (j // 10) * 0.2 - 0.9, -2.0), 1.0, 0.2 * j).matrix
        root["nodes"].append(dict(node, name=f"n{j}", matrix=[float(v) for v in np.asarray(m, np.float32).T.reshape(-1)]))
    root["scenes"][0]["nodes"] = list(range(90))
    root["buffers"][0]["uri"] = "data:application/octet-stream;base64," + base64.b64encode(binary).decode()
    path = tmp_path / "many.gltf"
    path.write_text(json.dumps(root))
    scene = load_scene(str(path))
    assert len(scene.primitives) == 1 and len(scene.bundles) == 90
    p = B.GaussianSplattingPlugin(0)
    try:
        sh = p.add_scene(scene)
        entities = sh.entities()
        assert len(sh.handles) == 1 and all(h is sh.handles[0] for h, _, _ in entities)
        img = p.render_entities_many(entities, VIEW)
        resident = SC.oracle_cloud(p.download(sh.handles[0]), "f32")
        oracle = [(resident, p.cloud_uniform(st, tr, h.aabb), False) for h, st, tr in entities]
        want = EO.frame(oracle, VIEW.to_abi(), [st.to_abi() for _, st, _ in entities], [st.num_classes for _, st, _ in entities])
        assert np.array_equal(p.sorted_entries(), want["sorted"])
        assert float(np.abs(img - want["image"]).max()) <= PIXEL_TOL
    finally:
        p.destroy()


# ---- 4. queued frames and ordering

def test_queued_frames_keep_their_tables():
    """Two back-to-back queued frames of 4097 and 300 entities, then bgs_sync: each is its synchronous frame."""
    p = B.GaussianSplattingPlugin(0)
    try:
        lists = []
        for k, seed in ((4097, 1), (300, 2)):
            n = 40 * k
            st = B.CloudSettings(aabb=bool(seed & 1))
            hw = p.add_cloud(SC.cloud_in_box(n, 400 + seed, half=1.6, scale=0.03, sh_degree=seed))
            u = p.cloud_uniform(st, SC.transform((0.05 * seed, 0.0, 0.0)), hw.aabb)
            parts = [p.subset(hw, ix) for ix in EM.pieces(n, k, seed)]
            lists.append(EM.Entities(p, parts, [u] * k, [st] * k, SV))
        sync = []
        for ents in lists:
            img = np.zeros((SV.height, SV.width, 4), np.float32)
            EM.ok(p, ents.call("many", img, abi.BGS_FORMAT_RGBA32F))
            sync.append(img)
        queued = [np.zeros((SV.height, SV.width, 4), np.float32) for _ in lists]
        for ents, img in zip(lists, queued):
            EM.ok(p, ents.call("many", img, abi.BGS_FORMAT_RGBA32F, abi.BGS_FLAG_ASYNC))
        assert p.sync()
        for a, b in zip(queued, sync):
            assert a.tobytes() == b.tobytes()
    finally:
        p.destroy()


def test_particle_step_between_queued_frames():
    """A cloud listed 1000 times: a particle step queued between two queued frames is seen by the second only."""
    p = B.GaussianSplattingPlugin(0)
    try:
        n, k = 400, 1000
        hw = p.add_cloud(SC.cloud_in_box(n, 5, centre=(0.0, 0.0, 0.0), half=0.1, scale=0.05, sh_degree=0))
        st = B.CloudSettings()
        trs = [SC.transform(((j % 40) * 0.09 - 1.8, 1.5 + (j // 40) * 0.06 - 0.75, -2.0), 1.0, 0.01 * j) for j in range(k)]
        ents = EM.Entities(p, [hw] * k, [p.cloud_uniform(st, tr, hw.aabb) for tr in trs], [st] * k, SV)
        behaviors = p.add_particles(random_particle_behaviors(n, 3))

        def frame(flags=0):
            img = np.zeros((SV.height, SV.width, 4), np.float32)
            EM.ok(p, ents.call("many", img, abi.BGS_FORMAT_RGBA32F, flags))
            return img

        before = frame()
        q1, q2 = np.zeros_like(before), np.zeros_like(before)
        EM.ok(p, ents.call("many", q1, abi.BGS_FORMAT_RGBA32F, abi.BGS_FLAG_ASYNC))
        p.step_particles(hw, behaviors, 0.25)
        EM.ok(p, ents.call("many", q2, abi.BGS_FORMAT_RGBA32F, abi.BGS_FLAG_ASYNC))
        assert p.sync()
        after = frame()
        assert q1.tobytes() == before.tobytes()
        assert q2.tobytes() == after.tobytes()
        assert before.tobytes() != after.tobytes()
    finally:
        p.destroy()


# ---- 5. refusals

def test_refusals_name_the_entity_and_keep_the_hooks():
    p = B.GaussianSplattingPlugin(0)
    try:
        n, k = 20000, 6000
        hw = p.add_cloud(SC.cloud_in_box(n, 9, half=1.6, scale=0.03, sh_degree=0))
        small = p.add_cloud(SC.cloud_in_box(50, 10, sh_degree=0))
        st = B.CloudSettings()
        u = p.cloud_uniform(st, None, hw.aabb)
        ents = EM.Entities(p, [small] * k, [p.cloud_uniform(st, None, small.aabb)] * k, [st] * k, SV)
        img = np.zeros((SV.height, SV.width, 4), np.float32)
        EM.ok(p, ents.call("many", img, abi.BGS_FORMAT_RGBA32F, abi.BGS_FLAG_NO_CHUNKS))
        want = capture(p, img, False)
        launches = p.last_launch_count
        sentinel = np.full((SV.height, SV.width, 4), 0.5, np.float32)
        pick = np.zeros((SV.height, SV.width), abi.PICK_DTYPE)

        def refused(call, match, k=None, frame=None, status=abi.BGS_EINVAL, e=ents, **kw):
            out = sentinel.copy()
            assert e.call(call, out, abi.BGS_FORMAT_RGBA32F, k=k, frame=frame, **kw) == status
            assert match in EM.error(p), EM.error(p)
            assert out.tobytes() == sentinel.tobytes()

        for call in ("many", "pick_many"):
            kw = dict(pick=pick) if call == "pick_many" else {}
            refused(call, "k = 0 is not in 1..65536", k=0, **kw)
            refused(call, "BGS_FLAG_SORT_ALL", frame=ents.frame(abi.BGS_FLAG_SORT_ALL), **kw)
            ents.clouds[4321] = None
            refused(call, "clouds[4321] is NULL", **kw)
            ents.clouds[4321] = small._h.value
            ents.ents[5000].rasterize_mode = 99
            refused(call, "entities[5000]: render: rasterize_mode 99", **kw)
            ents.ents[5000].rasterize_mode = int(M.Color)
            ents.ents[5000].draw_mode = 7
            refused(call, "entities[5000]: render: bad draw_mode", **kw)
            ents.ents[5000].draw_mode = 0
            ents.flags[5001] = 4
            refused(call, "entity_flags[5001]", **kw)
            ents.flags[5001] = 0
        over = EM.Entities(p, [hw] * abi.BGS_ENTITIES_MANY_MAX, [u] * abi.BGS_ENTITIES_MANY_MAX,
                           [st] * abi.BGS_ENTITIES_MANY_MAX, SV)
        refused("many", "must be < 2^30", e=over)
        refused("many", "k = 65537 is not in 1..65536", k=abi.BGS_ENTITIES_MANY_MAX + 1, e=over)
        refused("pick_many", "BGS_FLAG_ASYNC", frame=ents.frame(abi.BGS_FLAG_ASYNC), pick=pick)
        refused("pick_many", "out_pick is NULL")
        refused("many", "not ready", status=abi.BGS_NOT_READY, e=_NullView(ents))
        assert p.last_launch_count == launches
        _same(capture(p, img, False), want)
    finally:
        p.destroy()


class _NullView:
    """An Entities whose view is NULL (BGS_NOT_READY)."""

    def __init__(self, ents):
        self.e = ents

    def call(self, name, out, code, k=None, frame=None, **kw):
        e = self.e
        s = e.frame()
        return getattr(e.p._lib, "bgs_render_entities_" + name)(e.p._ctx, e.clouds, e.unis, e.ents, e.flags, e.k, None,
                                                                C.byref(s), None, None, out.ctypes.data, code, 0)


# ---- 6. the C++ host

CPP = r"""
#include <cstdio>
#include <fstream>
#include <vector>
#include "bgs.hpp"
// argv: cloud.bin (u64 n, then the four f32 planes), places.bin (u64 k, then k x 3 f32 translations), out.bin (the
// RGBA8 frame, then the pick frame, of render_entities_many / render_entities_pick_many at a 200 x 120 headless view)
int main(int argc, char** argv) {
    if (argc != 4) return 2;
    std::ifstream in(argv[1], std::ios::binary);
    uint64_t n = 0;
    in.read((char*)&n, 8);
    bgs::PlanarGaussian3d c;
    c.position_visibility.resize(n * 4); c.spherical_harmonic.resize(n * 48); c.rotation.resize(n * 4); c.scale_opacity.resize(n * 4);
    for (std::vector<float>* p : {&c.position_visibility, &c.spherical_harmonic, &c.rotation, &c.scale_opacity})
        in.read((char*)p->data(), p->size() * 4);
    std::ifstream pl(argv[2], std::ios::binary);
    uint64_t k = 0;
    pl.read((char*)&k, 8);
    std::vector<float> t(k * 3);
    pl.read((char*)t.data(), t.size() * 4);
    bgs::GaussianSplattingPlugin plugin(0);
    bgs::PlanarGaussian3dHandle h = plugin.add_cloud(c);
    std::vector<bgs::GaussianSplattingPlugin::SceneEntity> ents(k);
    for (uint64_t j = 0; j < k; ++j) {
        ents[j].cloud = &h;
        ents[j].transform.m[12] = t[3 * j]; ents[j].transform.m[13] = t[3 * j + 1]; ents[j].transform.m[14] = t[3 * j + 2];
    }
    const bgs_view view = bgs::headless_view(200, 120);
    std::vector<uint8_t> rgba(200 * 120 * 4), rgba2(rgba.size());
    std::vector<bgs_pick> pick(200 * 120);
    if (!plugin.render_entities_many(ents, view, rgba.data())) return 3;
    plugin.render_entities_pick_many(ents, view, rgba2.data(), pick.data());
    if (rgba2 != rgba) return 4;
    std::ofstream out(argv[3], std::ios::binary);
    out.write((const char*)rgba.data(), rgba.size());
    out.write((const char*)pick.data(), pick.size() * sizeof(bgs_pick));
    std::printf("k=%llu\n", (unsigned long long)k);
    return 0;
}
"""


def test_cpp_host_mirrors_match_python(tmp_path):
    import os
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    n, k = 300, 100
    cloud = SC.cloud_in_box(n, 12, centre=(0.0, 0.0, 0.0), half=0.1, scale=0.05)
    t = np.array([((j % 10) * 0.3 - 1.35, 1.5 + (j // 10) * 0.25 - 1.1, -2.0) for j in range(k)], np.float32)
    with open(tmp_path / "cloud.bin", "wb") as f:
        f.write(np.uint64(n).tobytes())
        for pl in (cloud.position_visibility, cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity):
            f.write(np.ascontiguousarray(pl, np.float32).tobytes())
    with open(tmp_path / "places.bin", "wb") as f:
        f.write(np.uint64(k).tobytes() + t.tobytes())
    src, exe = tmp_path / "many.cpp", tmp_path / "many"
    src.write_text(CPP)
    libdir = os.path.join(root, "bevy_gaussian_splatting_b200")
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-I", os.path.join(root, "include"), str(src), "-o", str(exe),
                    "-L", libdir, "-lbgs", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True, text=True)
    out = subprocess.run([str(exe), str(tmp_path / "cloud.bin"), str(tmp_path / "places.bin"), str(tmp_path / "out.bin")],
                         check=True, capture_output=True, text=True).stdout
    assert f"k={k}" in out
    got = (tmp_path / "out.bin").read_bytes()
    p = B.GaussianSplattingPlugin(0)
    try:
        h = p.add_cloud(cloud)
        trs = []
        for j in range(k):
            m = np.eye(4, dtype=np.float32)
            m[:3, 3] = t[j]
            trs.append(B.CloudTransform(m))
        ents = [(h, B.CloudSettings(), tr) for tr in trs]
        img = p.render_entities_many(ents, VIEW, fmt="rgba8_srgb")
        _, pick = p.render_entities_pick_many(ents, VIEW, fmt="rgba8_srgb")
        assert (pick["entity"][pick["entity"] != abi.BGS_PICK_NONE] > 63).any()
        assert got == img.tobytes() + pick.tobytes()
    finally:
        p.destroy()
