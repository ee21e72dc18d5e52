"""The bounding-box overlay (BGS_FLAG_VISUALIZE_BOUNDING_BOX) without a GPU: the entity oracle's edge decisions are the
literal VISUALIZE_BOUNDING_BOX branch of gaussian.wgsl on quad-uv, conic and surfel splats, at pixels within a few ulps
of the band edges and on them; its overlay walk draws only flagged entities' boxes and leaves unflagged frames as they
were; the host mirrors carry the setting."""
import numpy as np
import pytest

import bbox_cases as BX
import blend_cases as BC
import bevy_gaussian_splatting_b200 as B
import entity_cases as E
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import check_entities, check_scene_entities
from entity_oracle import entity_oracle as EO

GEOMS = ["obb3d", "obb2d", "aabb3d", "aabb2d"]


@pytest.mark.parametrize("geom", GEOMS)
def test_edge_decisions_are_the_wgsl_branch(oracle, geom):
    """Every (knife splat, target pixel) pair and every pair of the knife splats' bboxes: eo_edge_probe's covered pairs
    are edges exactly where the literal WGSL branch says so, on the uv the coverage decision used."""
    case = BX.band_case(oracle, geom, n_knife=64)
    s = case.settings
    u = B.GaussianSplattingPlugin.cloud_uniform(s)
    rec = oracle.project(case.cloud, case.view.to_abi(), u, s.to_abi(), case.knife_ids)
    # the knife pairs, then every pixel of each knife splat's bbox
    ids, pix = [case.knife_ids], [case.pixels]
    for i, r in zip(case.knife_ids, rec):
        xs, ys = np.meshgrid(np.arange(r["xlo"], r["xhi"] + 1), np.arange(r["ylo"], r["yhi"] + 1))
        ids.append(np.full(xs.size, i, np.uint32))
        pix.append(np.stack([xs.ravel(), ys.ravel()], 1))
    ids, pix = np.concatenate(ids), np.concatenate(pix)
    pos = np.searchsorted(case.knife_ids, ids)
    recs = rec[pos]
    xy = pix.astype(np.float32) + 0.5
    covered, edge, sxy = EO.edge_probe(recs, s.to_abi(), xy)
    pr = oracle.coverage_probe(recs, s.to_abi(), xy)
    assert np.array_equal(covered, pr["covered"] != 0)
    want, ws = BX.wgsl_visualize_bounding_box(*BX.probe_uv(pr, s.aabb))
    assert np.array_equal(edge, covered & want)
    assert np.array_equal(sxy[covered].view(np.uint32), ws[covered].view(np.uint32))
    # the knife pixels reach both thresholds, both axes and both sides, some of them within 2 ulps (or on it)
    k = len(case.knife_ids)
    sd, thr, on_x = BX.deciding_s(ws[:k])
    du = BC.ulps_from(sd, thr)
    assert covered[:k].all()
    near = np.abs(du) <= 4
    assert near.sum() >= 12, du
    assert (thr[near] == BX.LO).any() and (thr[near] == BX.HI).any()
    assert on_x[near].any() and (~on_x[near]).any()
    assert edge[:k][near].any() and (~edge[:k][near]).any()
    if s.aabb:   # m / R reaches the thresholds exactly (a quad-uv s at 0.08 moves in steps of 4 ulps there)
        assert (du == 0).any()
    # the knife pairs' edge decisions: the side of the threshold
    inside = np.where(thr == BX.LO, sd < thr, sd > thr)
    assert np.array_equal(edge[:k], inside | (edge[:k] & ~near))


def test_edge_rule_boundaries():
    """Around both band edges, uv one f32 ulp at a time: an edge exactly where s < 0.08f or s > 0.92f (s == 0.92f is
    reached and is not an edge); the same on the y axis; a NaN is not an edge."""
    for thr in (BX.LO, BX.HI):
        u0 = (thr - np.float32(0.5)) * np.float32(2.0)
        u = (np.array([u0], np.float32).view(np.int32) + np.arange(-40, 41, dtype=np.int32)).view(np.float32)
        edge, sv = BX.wgsl_visualize_bounding_box(u, np.zeros_like(u))
        sx = sv[:, 0]
        assert np.array_equal(edge, (sx < BX.LO) | (sx > BX.HI))
        assert edge.any() and (~edge).any()
        if thr == BX.HI:
            assert (sx == BX.HI).any() and not edge[sx == BX.HI].any()
        edge_y, _ = BX.wgsl_visualize_bounding_box(np.zeros_like(u), u)
        assert np.array_equal(edge_y, edge)
    nan = np.float32(np.nan)
    assert not BX.wgsl_visualize_bounding_box(np.array([nan]), np.array([np.float32(0.0)]))[0].any()


def test_frame_without_flags_is_eo_frame():
    """eo_frame_ex with no entity flag set is eo_frame, pixel for pixel, and draws no edge."""
    listed, view, sts = _kinds_entities()
    a = EO.frame(listed, view.to_abi(), [st.to_abi() for st in sts], [1] * len(sts))
    b = EO.frame(listed, view.to_abi(), [st.to_abi() for st in sts], [1] * len(sts), entity_flags=[0] * len(sts))
    assert a["image"].tobytes() == b["image"].tobytes()
    assert not b["edge_mask"].any()
    for key in ("sorted", "records", "tile_ranges", "tile_entries"):
        assert np.array_equal(a[key], b[key]), key


def test_only_flagged_entities_draw_boxes():
    """With entity j flagged, a pixel no edge reached is the unflagged frame's bit for bit (an edge only ends a walk
    early); with every entity flagged the edge mask is the union of the
    single-entity masks (a walk's first edge pair is one entity's)."""
    listed, view, sts = _kinds_entities()
    k = len(sts)
    none = EO.frame(listed, view.to_abi(), [st.to_abi() for st in sts], [1] * k, entity_flags=[0] * k)
    union = np.zeros_like(none["edge_mask"])
    for j in range(k):
        flags = [0] * k
        flags[j] = 1
        f = EO.frame(listed, view.to_abi(), [st.to_abi() for st in sts], [1] * k, entity_flags=flags)
        m = f["edge_mask"]
        assert m.any(), j
        assert f["image"][~m].tobytes() == none["image"][~m].tobytes()
        union |= m
    every = EO.frame(listed, view.to_abi(), [st.to_abi() for st in sts], [1] * k, entity_flags=[1] * k)
    assert np.array_equal(every["edge_mask"], union)


def _kinds_entities():
    """entity_cases' "kinds" room: quad-uv, conic and surfel 3D entities and the performer (quad-uv and conic)."""
    view = B.headless_view(200, 120)
    listed, sts = [], []
    for cloud, layout, tr, st in E.entities("kinds", n4=1500):
        u = B.GaussianSplattingPlugin.cloud_uniform(st, tr, _aabb(cloud))
        listed.append(E.oracle_entry(cloud, layout, u, st))
        sts.append(st)
    return listed, view, sts


def _aabb(cloud):
    p = cloud.position_visibility[:, :3]
    return (p.min(0), p.max(0))


def test_settings_carry_the_flag():
    assert B.CloudSettings(visualize_bounding_box=True).to_abi().flags & abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX
    assert not B.CloudSettings().to_abi().flags & abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX
    assert abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX == 64 and abi.BGS_ENTITY_VISUALIZE_BOUNDING_BOX == 1


def test_entities_may_differ_in_the_overlay_and_scenes_may_not():
    a, b = B.CloudSettings(), B.CloudSettings(visualize_bounding_box=True)
    assert check_entities([(None, a, None), (None, b, None)]) is a
    with pytest.raises(ValueError, match="visualize_bounding_box"):
        check_scene_entities([(None, a, None), (None, b, None)])
