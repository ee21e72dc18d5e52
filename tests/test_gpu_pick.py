"""bgs_render_entities_pick and bgs_cloud_select_in_view on the H100.  The pick call's colour frame is bgs_render_entities_ex's
byte for byte in every format and output mode, with and without a depth buffer and the overlays, on mixed-kind scenes with
a 4D performer, and its hooks are the one-round frame's; its pick frame matches pick_oracle's pairs under blend_cases'
bounds, with depths bit for bit the splat depths; the view selection is the set the entity oracle's records give; and
the refusals change nothing."""
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
FORMATS = {"f32": (np.float32, torch.float32, abi.BGS_FORMAT_RGBA32F), "f16": (np.float16, torch.float16, abi.BGS_FORMAT_RGBA16F),
           "u8": (np.uint8, torch.uint8, abi.BGS_FORMAT_RGBA8_SRGB)}


def _ok(p, rc):
    assert rc == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)


def _depth(seed):
    return torch.rand((H, W), generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda") * 0.04


class Scene:
    def __init__(self, p, listed, flags):
        self.p, self.flags = p, flags
        up = {}
        self.handles, self.unis, self.sts, self.counts, self.oracle = [], [], [], [], []
        for cloud, layout, tr, st in listed:
            if id(cloud) not in up:
                up[id(cloud)] = p.add_cloud(cloud, f16=layout in ("f16", "cov"), precompute_covariance=layout == "cov")
            h = up[id(cloud)]
            self.handles.append(h)
            self.unis.append(p.cloud_uniform(st, tr, h.aabb))
            self.sts.append(st)
            self.counts.append(len(cloud.position_visibility))
            self.oracle.append(E.oracle_entry(cloud, layout, self.unis[-1], st))

    def call(self, name, out, fmt, frame_flags=0, depth=None, device=False, pick=None):
        k = len(self.handles)
        s = self.sts[0].to_abi()
        s.flags = (s.flags & ~abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX) | frame_flags
        zd = None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * W)
        args = [self.p._ctx, (C.c_void_p * k)(*[h._h.value for h in self.handles]), (abi.bgs_cloud_uniform * k)(*self.unis),
                (abi.bgs_entity_settings * k)(*[entity_settings(st) for st in self.sts]), (C.c_uint32 * k)(*self.flags), k,
                C.byref(VIEW.to_abi()), C.byref(s), None, None if zd is None else C.byref(zd), _addr(out), FORMATS[fmt][2],
                int(device)]
        if name == "pick":
            args.append(_addr(pick))
        return getattr(self.p._lib, "bgs_render_entities_" + name)(*args)


def _addr(t):
    if t is None:
        return None
    return t.data_ptr() if isinstance(t, torch.Tensor) else t.ctypes.data


def _target(fmt, device, fill=None):
    npd, tod, _ = FORMATS[fmt]
    if device:
        t = torch.zeros((H, W, 4), dtype=tod, device="cuda")
        if fill is not None:
            t.copy_(torch.from_numpy(fill))
        return t
    return np.zeros((H, W, 4), npd) if fill is None else fill.copy()


def _pick_target(device):
    if device:
        return torch.full((H, W, 4), 0x7F7F7F7F, dtype=torch.int32, device="cuda")
    return np.full((H, W), 0x7F, np.uint8).repeat(16, axis=1).view(abi.PICK_DTYPE).reshape(H, W)


def _pick_host(t):
    if isinstance(t, torch.Tensor):
        torch.cuda.synchronize()
        return t.cpu().numpy().view(np.uint8).reshape(H, W, 16).view(abi.PICK_DTYPE).reshape(H, W)
    return t


def _bytes(t):
    if isinstance(t, torch.Tensor):
        torch.cuda.synchronize()
        return t.cpu().numpy().tobytes()
    return t.tobytes()


def _hooks(p):
    rec, ids = p.projected()
    return dict(stats=bytes(p.frame_stats()), sorted=p.sorted_entries().tobytes(), records=rec.tobytes(), ids=ids.tobytes(),
                ranges=p.tile_ranges().tobytes(), entries=p.tile_entries().tobytes())


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
