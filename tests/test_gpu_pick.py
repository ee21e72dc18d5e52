"""bgs_render_entities_pick and bgs_cloud_select_in_view on the H100.  The pick call's colour frame is bgs_render_entities_ex's
byte for byte in every format and output mode, with and without a depth buffer and the overlays, on mixed-kind scenes with
a 4D performer, and its hooks are the one-round frame's; its pick frame matches pick_oracle's pairs under blend_cases'
bounds (quad-uv, conic and surfel pairs), with depths bit for bit the splat depths; the view selection is the set the
entity oracle's records give; and the refusals change nothing."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

import bevy_gaussian_splatting_b200 as B
import blend_cases as BC
import entity_cases as E
import pick_cases as PK
import scene_cases as SC
import scene4d_cases as S4
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import entity_settings
from entity_oracle import entity_oracle as EO
from pick_oracle import pick_oracle as PO

pytestmark = pytest.mark.gpu

W, H = 200, 120   # (not tile multiples)
VIEW = B.headless_view(W, H)
FORMATS = PK.FORMATS
_ok, _addr, _bytes, _hooks = PK.ok, PK.addr, PK.as_bytes, PK.hooks


def _depth(seed):
    return torch.rand((H, W), generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda") * 0.04


def Scene(p, listed, flags):
    return PK.Scene(p, listed, flags, VIEW)


def _target(fmt, device, fill=None):
    return PK.target(VIEW, fmt, device, fill)


def _pick_target(device):
    return PK.pick_target(VIEW, device)


def _pick_host(t):
    return PK.pick_host(t, VIEW)


OVERLAYS = {"none": (0, None), "frame": (abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX, None), "entity": (0, (1, 0, 0, 1, 0, 1))}


@pytest.mark.parametrize("case", ["kinds", "surfel_4d"])
@pytest.mark.parametrize("with_depth", [False, True])
@pytest.mark.parametrize("overlay", list(OVERLAYS))
def test_pick_colour_is_entities_ex_and_depths_are_splat_depths(case, with_depth, overlay):
    frame_flags, eflags = OVERLAYS[overlay]
    listed = E.entities(case)
    flags = list(eflags or [0] * len(listed))
    depth = _depth(5) if with_depth else None
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Scene(p, listed, flags)
        modes = {"plain": 0, "premul": abi.BGS_FLAG_PREMULTIPLIED_OUT, "over": abi.BGS_FLAG_BLEND_OVER_TARGET}
        rng = np.random.default_rng(3)
        for fmt in FORMATS:
            for device in (False, True):
                for mode, mflag in modes.items():
                    if mode == "over" and not device:
                        continue   # (host blend-over reads the context's last frame: covered by the device target)
                    fill = None
                    if mode == "over":
                        fill = (rng.random((H, W, 4)) * (255 if fmt == "u8" else 1)).astype(FORMATS[fmt][0])
                    out, pick = _target(fmt, device, fill), _pick_target(device)
                    _ok(p, sc.call("pick", out, fmt, frame_flags | mflag | abi.BGS_FLAG_CHUNKS, depth, device, pick))
                    torch.cuda.synchronize()
                    got = _hooks(p)
                    sd = p.splat_depths()
                    launches = p.last_launch_count
                    want = _target(fmt, device, fill)
                    _ok(p, sc.call("ex", want, fmt, frame_flags | mflag | abi.BGS_FLAG_NO_CHUNKS, depth, device))
                    assert _bytes(out) == _bytes(want), (fmt, device, mode)
                    torch.cuda.synchronize()
                    want_hooks = _hooks(p)
                    for key in want_hooks:
                        assert got[key] == want_hooks[key], key
                    assert launches == p.last_launch_count + (0 if with_depth else 1)
                    # depths: the splat depth of the picked rank, bit for bit
                    pk = _pick_host(pick)
                    _, ids = p.projected()
                    rank = PK.to_rank(pk, ids, sc.counts)
                    some = rank >= 0
                    assert some.mean() > 0.2
                    assert np.array_equal(pk["depth"][some].view(np.uint32), sd[rank[some]].view(np.uint32))
                    # (a pair whose alpha underflows blends with w = 0: it is picked where nothing else blends)
                    assert (pk["weight"][some] >= 0).all() and (pk["weight"][some] <= 1).all()
                    if with_depth:
                        assert np.array_equal(sd.view(np.uint32), p.splat_depths().view(np.uint32))
    finally:
        p.destroy()


@pytest.mark.parametrize("with_depth", [False, True])
@pytest.mark.parametrize("overlay", ["none", "entity"])
@pytest.mark.parametrize("saturated", [False, True])
def test_pick_matches_the_pick_oracle(with_depth, overlay, saturated):
    listed = PK.oracle_scene()
    if saturated:   # opaque splats: most pixels stop early
        listed = [(c, l, tr, dataclasses.replace(st, global_opacity=1.0, global_scale=2.5)) for c, l, tr, st in listed]
    flags = [1, 0, 1] if overlay == "entity" else [0, 0, 0]
    depth = _depth(9) if with_depth else None
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Scene(p, listed, flags)
        out, pick = _target("f32", False), _pick_target(False)
        _ok(p, sc.call("pick", out, "f32", 0, depth, False, pick))
        want = EO.frame(sc.oracle, VIEW.to_abi(), [st.to_abi() for st in sc.sts], [1] * len(sc.sts),
                        scene=None if depth is None else depth.cpu().numpy(), entity_flags=flags)
        _, ids = p.projected()
        assert np.array_equal(ids, want["rank_to_id"])
        kinds = PK.rank_kinds(want["rank_to_id"], sc.counts, sc.sts, flags)
        pairs = PO.pairs(want, kinds, W, H, BC.alpha_error_coefs(False), scene=None if depth is None else depth.cpu().numpy())
        # conic alphas take the USE_AABB coefficients: use the larger of the two per pair
        c_aabb = BC.alpha_error_coefs(True)
        pairs_aabb = PO.pairs(want, kinds, W, H, c_aabb, scene=None if depth is None else depth.cpu().numpy())
        pairs["bound"] = np.maximum(pairs["bound"], pairs_aabb["bound"])
        rank = PK.to_rank(pick, ids, sc.counts)
        picked, strict = PK.check_pick(pick, rank, pairs)
        assert picked > 0.2 * W * H and strict > 0.5 * picked, (picked, strict)
        some = rank >= 0
        assert np.array_equal(pick["depth"][some].view(np.uint32), want["depths"][rank[some]].view(np.uint32))
        # the same cloud listed twice: both entities picked somewhere, with the same index space
        ents = set(np.unique(pick["entity"][some]).tolist())
        assert {0, 2} <= ents, ents
        if with_depth:   # a splat behind the scene's depth at a pixel is never picked there
            zs = depth.cpu().numpy()
            assert (pick["depth"][some] >= zs[some]).all()
        if overlay == "entity":   # edge pixels of an entity with its overlay: w = T
            assert want["edge_mask"].any()
    finally:
        p.destroy()


def _surfel_scene(name):
    """2DGS aabb surfels alone, beside quad-uv and conic entities, and entity_cases' surfel_4d case."""
    if name == "surfel_4d":
        return E.entities("surfel_4d")
    room = S4.room()
    surf = dict(gaussian_mode=B.GaussianMode.Gaussian2d, aabb=True)
    (c0, l0, _, tr0, kw0), (c1, l1, _, tr1, kw1), (c2, l2, _, tr2, kw2), (c3, l3, _, tr3, kw3) = room
    if name == "surfels":
        return [(c0, l0, tr0, B.CloudSettings(**kw0, **surf)), (c1, l1, tr1, B.CloudSettings(**kw1, **surf)),
                (c3, l3, tr3, B.CloudSettings(**kw3, **surf)),
                (c0, l0, SC.transform((0.5, 0.2, -0.6), 0.9, 0.4), B.CloudSettings(global_opacity=0.7, **surf))]
    return [(c0, l0, tr0, B.CloudSettings(**kw0, **surf)), (c1, l1, tr1, B.CloudSettings(**kw1)),
            (c2, l2, tr2, B.CloudSettings(**kw2, aabb=True)), (c3, l3, tr3, B.CloudSettings(**kw3, **surf))]


@pytest.mark.parametrize("with_depth", [False, True])
@pytest.mark.parametrize("overlay", ["none", "entity"])
@pytest.mark.parametrize("scene", ["surfels", "surfel_quad_conic", "surfel_4d"])
def test_pick_matches_the_pick_oracle_on_surfels(scene, with_depth, overlay):
    """Surfel pairs held to pick_oracle's restatement of the surfel branch (surfel alphas come from __expf, as conic
    ones do: alpha_error_coefs(True)), beside quad-uv and conic ones and in the surfel_4d entity case."""
    listed = _surfel_scene(scene)
    flags = [(j + 1) % 2 if overlay == "entity" else 0 for j in range(len(listed))]
    depth = _depth(13) if with_depth else None
    zs = None if depth is None else depth.cpu().numpy()
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Scene(p, listed, flags)
        out, pick = _target("f32", False), _pick_target(False)
        _ok(p, sc.call("pick", out, "f32", 0, depth, False, pick))
        want = EO.frame(sc.oracle, VIEW.to_abi(), [st.to_abi() for st in sc.sts], [1] * len(sc.sts), scene=zs,
                        entity_flags=flags)
        _, ids = p.projected()
        assert np.array_equal(ids, want["rank_to_id"])
        kinds = PK.rank_kinds(want["rank_to_id"], sc.counts, sc.sts, flags)
        assert ((kinds & 3) == 2).sum() > 1000
        pairs = PO.pairs(want, kinds, W, H, BC.alpha_error_coefs(True), scene=zs)
        if scene != "surfels":   # quad-uv pairs: the larger of the two bounds
            pairs_obb = PO.pairs(want, kinds, W, H, BC.alpha_error_coefs(False), scene=zs)
            pairs["bound"] = np.maximum(pairs["bound"], pairs_obb["bound"])
        rank = PK.to_rank(pick, ids, sc.counts)
        picked, strict = PK.check_pick(pick, rank, pairs)
        assert picked > 0.1 * W * H and strict > 0.3 * picked, (picked, strict)
        # surfels are picked, and strictly decided somewhere
        some = rank >= 0
        assert ((kinds[rank[some]] & 3) == 2).sum() > 0.05 * W * H
        assert np.array_equal(pick["depth"][some].view(np.uint32), want["depths"][rank[some]].view(np.uint32))
        if with_depth:
            assert (pick["depth"][some] >= zs[some]).all()
        if overlay == "entity":
            assert want["edge_mask"].any()
    finally:
        p.destroy()


def test_pick_empty_tiles_and_refusals():
    listed = PK.oracle_scene()[:1]
    cloud = listed[0][0]
    far = SC.transform((0.0, 0.0, 500.0))   # everything behind the camera: every tile empty
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Scene(p, [(cloud, "f32", far, B.CloudSettings())], [0])
        out, pick = _target("f32", True), _pick_target(True)
        _ok(p, sc.call("pick", out, "f32", abi.BGS_FLAG_BLEND_OVER_TARGET, None, True, pick))
        pk = _pick_host(pick)
        assert (pk["entity"] == abi.BGS_PICK_NONE).all() and (pk["index"] == abi.BGS_PICK_NONE).all()
        assert (pk["weight"] == 0).all() and (pk["depth"] == 0).all()
        # refusals: nothing written, hooks kept
        sc = Scene(p, listed, [0])
        _ok(p, sc.call("pick", _target("f32", False), "f32", 0, None, False, _pick_target(False)))
        before = _hooks(p)
        buf = torch.zeros(H * W * 4 + 4, dtype=torch.int32, device="cuda")
        for flags, device, pick_ptr in ((0, False, None), (abi.BGS_FLAG_ASYNC, False, _pick_target(False).ctypes.data),
                                        (0, True, buf.data_ptr() + 8)):
            out = _target("f32", device)
            o0 = _bytes(out)
            assert _call_raw(sc, out, pick_ptr, flags, device) == abi.BGS_EINVAL, (flags, device)
            assert _bytes(out) == o0
        assert _hooks(p) == before
        with pytest.raises(ValueError):
            p.render_entities_pick([], VIEW)
    finally:
        p.destroy()


def _call_raw(sc, out, pick_ptr, flags, device):
    k = len(sc.handles)
    s = sc.sts[0].to_abi()
    s.flags |= flags
    return sc.p._lib.bgs_render_entities_pick(sc.p._ctx, (C.c_void_p * k)(*[h._h.value for h in sc.handles]),
                                              (abi.bgs_cloud_uniform * k)(*sc.unis),
                                              (abi.bgs_entity_settings * k)(*[entity_settings(st) for st in sc.sts]), None, k,
                                              C.byref(VIEW.to_abi()), C.byref(s), None, None, _addr(out),
                                              abi.BGS_FORMAT_RGBA32F, int(device), None if pick_ptr is None else C.c_void_p(pick_ptr))


def _view_set(cloud, layout, u, mask, view=VIEW):
    """The gaussians inside by the entity oracle's records: in the frustum (listed), centre in the frame, mask set."""
    st = B.CloudSettings()
    want = EO.frame([E.oracle_entry(cloud, layout, u, st)], view.to_abi(), [st.to_abi()], [1], want_image=False)
    cx, cy = want["records"][:, 0], want["records"][:, 1]
    ok = (cx >= 0) & (cx < view.width) & (cy >= 0) & (cy < view.height)
    ids = want["rank_to_id"][ok]
    hit = mask[np.floor(cy[ok]).astype(np.int64), np.floor(cx[ok]).astype(np.int64)] != 0
    inside = np.zeros(len(cloud.position_visibility), bool)
    inside[ids[hit]] = True
    return inside


@pytest.mark.parametrize("which", [0, 1, 2, 3])   # f32 SH 3, f16 SH 1, covariance, f32 SH 0
@pytest.mark.parametrize("device_mask", [False, True])
def test_select_in_view_matches_the_oracle(which, device_mask):
    cloud, layout, _, tr, _ = S4.room()[which]
    rng = np.random.default_rng(which)
    masks = {"random": rng.random((H, W)) < 0.5, "rect": np.zeros((H, W), bool)}
    masks["rect"][20:90, 40:150] = True
    p = B.GaussianSplattingPlugin(0)
    try:
        h = p.add_cloud(cloud, f16=layout in ("f16", "cov"), precompute_covariance=layout == "cov")
        for tname, t in (("identity", None), ("transform", tr)):
            for mname, mask in masks.items():
                want = _view_set(cloud, layout, p.cloud_uniform(B.CloudSettings(), t, h.aabb), mask)
                assert 0 < want.sum() < len(want)
                m = torch.from_numpy(mask.astype(np.uint8)).cuda() if device_mask else mask
                n = p.select_in_view(h, VIEW, m, transform=t, mode="replace")
                vis = p.visibility(h)
                assert n == want.sum(), (tname, mname)
                assert np.array_equal(vis == 1.0, want) and np.array_equal(vis == 0.0, ~want), (tname, mname)
                # ADD: the union with what was there
                base = (rng.random(len(want)) < 0.3).astype(np.float32)
                p.set_visibility(h, base)
                n = p.select_in_view(h, VIEW, m, transform=t, mode="add")
                assert n == want.sum()
                assert np.array_equal(p.visibility(h), np.where(want, np.float32(1), base))
        # culled gaussians are never selected, whatever the mask: everything behind the camera
        assert p.select_in_view(h, VIEW, np.ones((H, W), bool), transform=SC.transform((0, 0, 500.0))) == 0
        assert (p.visibility(h) == 0).all()
        # refusals change nothing
        p.set_visibility(h, np.full(len(cloud.position_visibility), 0.25, np.float32))
        lane = p.visibility(h).tobytes()
        u, v = p.cloud_uniform(B.CloudSettings(), None, h.aabb), VIEW.to_abi()
        mk = np.ones((H, W), np.uint8)
        lib, ctx = p._lib, p._ctx
        assert lib.bgs_cloud_select_in_view(ctx, h._h, C.byref(u), C.byref(v), mk.ctypes.data, 0, 7, None) == abi.BGS_EINVAL
        assert lib.bgs_cloud_select_in_view(ctx, h._h, C.byref(u), C.byref(v), None, 0, 0, None) == abi.BGS_EINVAL
        assert lib.bgs_cloud_select_in_view(ctx, h._h, None, C.byref(v), mk.ctypes.data, 0, 0, None) == abi.BGS_EINVAL
        assert lib.bgs_cloud_select_in_view(ctx, h._h, C.byref(u), None, mk.ctypes.data, 0, 0, None) == abi.BGS_EINVAL
        assert lib.bgs_cloud_select_in_view(ctx, None, C.byref(u), C.byref(v), mk.ctypes.data, 0, 0, None) == abi.BGS_EINVAL
        assert lib.bgs_cloud_select_in_view(None, h._h, C.byref(u), C.byref(v), mk.ctypes.data, 0, 0, None) == abi.BGS_EINVAL
        assert lib.bgs_cloud_select_in_view(ctx, h._h, C.byref(u), C.byref(v), mk.ctypes.data, 1, 0, None) == abi.BGS_EINVAL
        assert p.visibility(h).tobytes() == lane
    finally:
        p.destroy()


def test_select_in_view_refuses_4d():
    perf = S4.performer(500, 2)
    p = B.GaussianSplattingPlugin(0)
    try:
        h = p.add_cloud(perf)
        lane = p.visibility(h).tobytes()
        u, v = p.cloud_uniform(B.CloudSettings(), None, h.aabb), VIEW.to_abi()
        mk = np.ones((H, W), np.uint8)
        assert p._lib.bgs_cloud_select_in_view(p._ctx, h._h, C.byref(u), C.byref(v), mk.ctypes.data, 0, 0, None) == abi.BGS_EINVAL
        assert p.visibility(h).tobytes() == lane
    finally:
        p.destroy()


def test_select_picked_is_the_host_set_of_the_pick_frame():
    listed = PK.oracle_scene()
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = Scene(p, listed, [0, 0, 0])
        ents = [(h, st, tr) for h, st, (_, _, tr, _) in zip(sc.handles, sc.sts, listed)]
        rgba, pick = p.render_entities_pick(ents, VIEW)
        mask = np.zeros((H, W), bool)
        mask[30:80, 50:160] = True
        n = p.select_picked(ents, pick, mask, min_weight=0.05)
        sel = mask & (pick["entity"] != abi.BGS_PICK_NONE) & (pick["weight"] >= np.float32(0.05))
        total = 0
        for h in {id(h): h for h in sc.handles}.values():
            js = [j for j, e in enumerate(sc.handles) if e is h]
            want = np.zeros(h.n, bool)
            want[pick["index"][sel & np.isin(pick["entity"], js)]] = True
            total += want.sum()
            assert np.array_equal(p.visibility(h) == 1.0, want)
        assert n == total > 0
        # the colour frame is render_entities' frame
        assert rgba.tobytes() == p.render_entities(ents, VIEW).tobytes()
    finally:
        p.destroy()
