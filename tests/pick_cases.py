"""Inputs and checks of bgs_render_entities_pick's and bgs_cloud_select_in_view's tests (tests/test_gpu_pick.py,
tests/test_host_pick.py): entity_cases' room and performer, a quad-uv + conic scene with one cloud listed twice, and the
pick frame against pick_oracle's pairs under blend_cases' per-alpha error bounds."""
from __future__ import annotations

import numpy as np

import bevy_gaussian_splatting_b200 as B
import blend_cases as BC
import scene_cases as SC
import scene4d_cases as S4
from bevy_gaussian_splatting_b200 import abi

M, G = B.RasterizeMode, B.GaussianMode


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
