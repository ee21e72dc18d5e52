"""pick_oracle's surfel restatement without a GPU: on every pixel around every visible surfel of the 2DGS aabb cases of
blend_cases and bbox_cases, the pick oracle's coverage and edge decisions (raster.cu's surfel branch, restated on the
surfel extras eo_frame_ex exports) are the entity oracle's own (decide() and box_edge() on its splat records), and the
exported extras are the entity oracle's records' own bits."""
import dataclasses

import numpy as np
import pytest

import bbox_cases as BX
import blend_cases as BC
import bevy_gaussian_splatting_b200 as B
from entity_oracle import entity_oracle as EO
from pick_oracle import pick_oracle as PO

MARGIN = 2   # pixels probed beyond each surfel's bbox (where coverage must fail)


def _case(oracle, which):
    """(cloud, view, settings) of one 2DGS aabb case."""
    if which == "band":
        c = BX.band_case(oracle, "aabb2d", n_knife=64)
    elif which == "saturated":
        return BC.saturated_case("aabb2d")
    else:
        c = BC.knife_case(oracle, "aabb2d", which == "knife_saturated")
    return c.cloud, c.view, c.settings


@pytest.mark.parametrize("which", ["band", "knife", "knife_saturated", "saturated"])
def test_surfel_decisions_are_the_entity_oracles(oracle, which):
    cloud, view, s = _case(oracle, which)
    assert s.aabb and s.gaussian_mode == B.GaussianMode.Gaussian2d
    u = B.GaussianSplattingPlugin.cloud_uniform(s)
    fr = EO.frame([(cloud, u, False)], view.to_abi(), [s.to_abi()], [1], entity_flags=[1], want_image=False)
    rec, ex, ids = fr["records"], fr["surfel_extra"], fr["rank_to_id"]
    splats = oracle.project(cloud, view.to_abi(), u, s.to_abi(), ids)
    # the exported extras: the entity oracle's surfel record fields, bit for bit (e1..e3's w lanes are 0)
    want_ex = np.zeros((len(ids), 16), np.float32)
    want_ex[:, 0:4] = splats["extra"][:, 3:7]
    for q in range(3):
        want_ex[:, 4 * (q + 1):4 * (q + 1) + 3] = splats["extra"][:, 7 + 3 * q:10 + 3 * q]
    assert np.array_equal(ex.view(np.uint32), want_ex.view(np.uint32))
    # every pixel of each drawn surfel's bbox and MARGIN around it
    W, H = view.width, view.height
    r_all, xy_all = [], []
    for r, sp in enumerate(splats):
        if sp["xlo"] > sp["xhi"] or sp["ylo"] > sp["yhi"]:
            continue
        xs = np.arange(max(sp["xlo"] - MARGIN, 0), min(sp["xhi"] + MARGIN, W - 1) + 1)
        ys = np.arange(max(sp["ylo"] - MARGIN, 0), min(sp["yhi"] + MARGIN, H - 1) + 1)
        gx, gy = np.meshgrid(xs, ys)
        r_all.append(np.full(gx.size, r, np.int64))
        xy_all.append(np.stack([gx.ravel(), gy.ravel()], 1))
    r_all, xy = np.concatenate(r_all), np.concatenate(xy_all).astype(np.float32) + np.float32(0.5)
    covered, edge = PO.surfel_probe(rec[r_all], ex[r_all], xy)
    want_cov, want_edge, _ = EO.edge_probe(splats[r_all], s.to_abi(), xy)
    assert np.array_equal(covered, want_cov), np.flatnonzero(covered != want_cov)[:10]
    assert np.array_equal(edge, want_edge), np.flatnonzero(edge != want_edge)[:10]
    # both decisions go both ways
    assert covered.any() and (~covered).any() and edge.any() and (covered & ~edge).any()


def test_pick_pairs_of_a_surfel_frame_blend_like_the_entity_oracle(oracle):
    """pick_oracle's pairs of a surfel frame: at every pixel, the f64 colour sum of its pairs' w times the record colour
    is the entity oracle's f32 image within the pairs' bounds."""
    cloud, view, s = BC.saturated_case("aabb2d")
    s = dataclasses.replace(s, global_opacity=0.4)
    u = B.GaussianSplattingPlugin.cloud_uniform(s)
    fr = EO.frame([(cloud, u, False)], view.to_abi(), [s.to_abi()], [1], entity_flags=[0])
    kinds = np.full(fr["n_vis"], 2, np.uint8)
    pr = PO.pairs(fr, kinds, view.width, view.height, BC.alpha_error_coefs(True))
    off, rank, w, bd = pr["offsets"].astype(np.int64), pr["rank"], pr["w"], pr["bound"]
    pix = np.repeat(np.arange(view.width * view.height), np.diff(off))
    rgb = fr["records"][rank, 8:11].astype(np.float64)
    got = np.zeros((view.width * view.height, 3))
    np.add.at(got, pix, w[:, None] * rgb)
    err = np.zeros(view.width * view.height)
    np.add.at(err, pix, bd * np.abs(rgb).max(1))
    img = fr["image"].reshape(-1, 4)[:, :3].astype(np.float64)
    assert (np.diff(off) > 0).sum() > 0.3 * view.width * view.height
    # (the entity oracle blends in f32: its own rounding adds a few ulps per pair)
    slack = 1e-5 * (np.diff(off) + 1)
    assert (np.abs(got - img).max(1) <= err + slack).all()
