"""Inputs and checks of bgs_render_entities_pick's and bgs_cloud_select_in_view's tests (tests/test_gpu_pick.py,
tests/test_gpu_pick_paths.py, tests/test_host_pick.py): entity_cases' room and performer, a quad-uv + conic scene with one
cloud listed twice, the pick frame against pick_oracle's pairs under blend_cases' per-alpha error bounds, and the entity
list / target helpers the GPU tests call bgs_render_entities_ex and _pick through."""
from __future__ import annotations

import ctypes as C

import numpy as np

import bevy_gaussian_splatting_b200 as B
import blend_cases as BC
import entity_cases as E
import scene_cases as SC
import scene4d_cases as S4
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import entity_settings

M, G = B.RasterizeMode, B.GaussianMode

# name -> (numpy dtype, torch dtype name, BGS_FORMAT_*)
FORMATS = {"f32": (np.float32, "float32", abi.BGS_FORMAT_RGBA32F), "f16": (np.float16, "float16", abi.BGS_FORMAT_RGBA16F),
           "u8": (np.uint8, "uint8", abi.BGS_FORMAT_RGBA8_SRGB)}
MODES = {"plain": 0, "premul": abi.BGS_FLAG_PREMULTIPLIED_OUT, "over": abi.BGS_FLAG_BLEND_OVER_TARGET}


def ok(p, rc):
    assert rc == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)


def addr(t):
    if t is None:
        return None
    return t.ctypes.data if isinstance(t, np.ndarray) else t.data_ptr()


class Scene:
    """An entity list [(cloud, layout, transform, CloudSettings)] uploaded into plugin `p` (a cloud listed twice is uploaded
    once), with one entity-flags word per entity, called through bgs_render_entities_ex / _pick at `view`.  The frame's
    settings are entity 0's, without the frame-wide overlay bit, | frame_flags."""

    def __init__(self, p, listed, flags, view):
        self.p, self.flags, self.view = p, flags, view
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
        zd = None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * self.view.width)
        args = [self.p._ctx, (C.c_void_p * k)(*[h._h.value for h in self.handles]), (abi.bgs_cloud_uniform * k)(*self.unis),
                (abi.bgs_entity_settings * k)(*[entity_settings(st) for st in self.sts]),
                (C.c_uint32 * k)(*self.flags), k, C.byref(self.view.to_abi()), C.byref(s), None,
                None if zd is None else C.byref(zd), addr(out), FORMATS[fmt][2], int(device)]
        if name == "pick":
            args.append(addr(pick))
        return getattr(self.p._lib, "bgs_render_entities_" + name)(*args)


def target(view, fmt, device, fill=None):
    """A colour target of `view` in `fmt`: zeros, or a copy of `fill`; a torch tensor on the GPU when `device`."""
    npd = FORMATS[fmt][0]
    if device:
        import torch

        t = torch.zeros((view.height, view.width, 4), dtype=getattr(torch, FORMATS[fmt][1]), device="cuda")
        if fill is not None:
            t.copy_(torch.from_numpy(fill))
        return t
    return np.zeros((view.height, view.width, 4), npd) if fill is None else fill.copy()


def pick_target(view, device):
    """A pick target of `view`, every byte 0x7F (so a record the call leaves unwritten shows)."""
    H, W = view.height, view.width
    if device:
        import torch

        return torch.full((H, W, 4), 0x7F7F7F7F, dtype=torch.int32, device="cuda")
    return np.full((H, W), 0x7F, np.uint8).repeat(16, axis=1).view(abi.PICK_DTYPE).reshape(H, W)


def pick_host(t, view):
    if isinstance(t, np.ndarray):
        return t
    import torch

    torch.cuda.synchronize()
    return t.cpu().numpy().view(np.uint8).reshape(view.height, view.width, 16).view(abi.PICK_DTYPE).reshape(view.height, view.width)


def as_bytes(t):
    if isinstance(t, np.ndarray):
        return t.tobytes()
    import torch

    torch.cuda.synchronize()
    return t.cpu().numpy().tobytes()


def hooks(p):
    """The last frame's debug hooks and stats, as bytes."""
    rec, ids = p.projected()
    return dict(stats=bytes(p.frame_stats()), sorted=p.sorted_entries().tobytes(), records=rec.tobytes(), ids=ids.tobytes(),
                ranges=p.tile_ranges().tobytes(), entries=p.tile_entries().tobytes())


def oracle_scene():
    """[(cloud, layout, transform, CloudSettings)]: quad-uv and conic entities only (the kinds pick_oracle restates), the
    f32 room cloud listed twice with different transforms (same index, different entity)."""
    room = S4.room()
    (c0, l0, _, tr0, kw0), (c1, l1, _, tr1, kw1) = room[0], room[1]
    return [(c0, l0, tr0, B.CloudSettings(**kw0)),
            (c1, l1, tr1, B.CloudSettings(**kw1, aabb=True)),
            (c0, l0, SC.transform((0.5, 0.2, -0.6), 0.9, 0.4), B.CloudSettings(global_opacity=0.7, aabb=True))]


def rank_kinds(rank_to_id, counts, sts, flags):
    """Each rank's kind byte: its entity's blend kind (0 quad-uv, 1 conic, 2 surfel) | 4 when the entity draws its boxes."""
    offs = np.cumsum([0] + list(counts))
    ent = np.searchsorted(offs, rank_to_id, side="right") - 1
    kind = np.array([0 if not st.aabb else (2 if st.gaussian_mode == G.Gaussian2d else 1) for st in sts], np.uint8)
    box = np.array([4 if f else 0 for f in flags], np.uint8)
    return (kind | box)[ent]


def to_rank(pick, rank_to_id, counts):
    """Each pixel's picked rank (-1 where nothing blends), through the global index offset[entity] + index."""
    offs = np.cumsum([0] + list(counts)).astype(np.int64)
    inv = np.full(int(offs[-1]), -1, np.int64)
    inv[rank_to_id] = np.arange(len(rank_to_id))
    none = pick["entity"] == abi.BGS_PICK_NONE
    g = np.where(none, 0, offs[np.minimum(pick["entity"], len(counts) - 1)] + pick["index"])
    return np.where(none, -1, inv[g])


def check_pick(pick, rank, pairs, near_stop_slack: float = 1.01 * BC.T_STOP):
    """The pick frame against pick_oracle's pairs: NONE exactly where the oracle blends nothing; where the oracle's best
    weight beats every other pair's by more than both bounds, the same pair; elsewhere a pair whose oracle weight is within
    bounds of the maximum; the weight within bounds of the oracle's w for that pair.  At near-stop pixels the kernel may
    blend one pair more or less, whose weight is below ~T_STOP.  Returns (pixels with a pick, pixels decided strictly)."""
    H, W = pick.shape
    off, pr, pw, pb = pairs["offsets"], pairs["rank"], pairs["w"], pairs["bound"]
    near = pairs["near_stop"].reshape(-1)
    flat_rank, flat_w = rank.reshape(-1), pick["weight"].reshape(-1).astype(np.float64)
    picked = strict = 0
    for pix in range(H * W):
        a, b = int(off[pix]), int(off[pix + 1])
        if a == b:
            assert flat_rank[pix] == -1 and flat_w[pix] == 0.0, pix
            assert pick["depth"].reshape(-1)[pix] == 0.0, pix
            continue
        if flat_rank[pix] == -1:
            assert near[pix] and b - a == 1 and pw[a] <= near_stop_slack, pix
            continue
        picked += 1
        r, w, bd = pr[a:b], pw[a:b], pb[a:b]
        hit = np.flatnonzero(r == flat_rank[pix])
        if hit.size == 0:   # (a pair past the oracle's stop)
            assert near[pix] and flat_w[pix] <= near_stop_slack + 1e-6, pix
            continue
        j = int(hit[0])
        assert abs(flat_w[pix] - w[j]) <= bd[j] + 1e-12, (pix, flat_w[pix], w[j], bd[j])
        best = int(np.argmax(w))
        others = np.delete(np.arange(b - a), best)
        margin = bd[best] + (bd[others] if others.size else 0.0)
        extra = near_stop_slack if near[pix] else 0.0
        if np.all(w[best] - (w[others] if others.size else -1.0) > margin + extra):
            strict += 1
            assert j == best, (pix, j, best)
        else:
            assert w[j] >= w[best] - bd[best] - bd[j] - extra, pix
    return picked, strict
