"""The oracle's coverage probe and blend trace, and the blend constructions of tests/blend_cases.py (no GPU).

* Every construction reaches the pair classes it claims, with a stated minimum count per class.
* `coverage_probe` makes exactly the decisions and alphas `render_tiles` blends with, and `blend_trace`'s f32 walk stops
  where `render_tiles` stops: an f32 replay of the trace's decisions reproduces the tile_mode image bit for bit.
* The oracle's own f32 tile_mode image lies within the per-pixel bound of the trace's float64 blend (with the bound's
  USE_OBB / USE_AABB alpha term, which the oracle's libm exp meets with room), so the bound used on the GPU frames is
  neither vacuous nor broken before a GPU is involved."""
import time

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import blend_cases as BC

# per (geometry, saturated, heavy): minimum count of each class its knife-edge frame reaches.  Counts at these seeds:
#   obb3d            ~30 K0, 31 K+, 10-13 K-, 5-9 KF, 51 KS, 3 + 3 KCH, 10-12 even, 9-10 odd, 10 tail, 1-2 KF at each
#                    position, 59 + 18 KPX, 77 in later rounds
#   obb3d heavy      the same but for the list positions (the big background splats are in every warp's list): 20-22 even
#   aabb3d           35-40 K0, 10-18 K+, 11-13 K-, ~50 KS
#   aabb2d / obb2d   surfel scales fit less tightly: 1-7 of each K class; obb2d 3-6 even, 8-10 odd, 6-9 tail.  Surfel
#                    OBB records have uy = vx = 0, so u = ux dx either way: no fma split exists there.
OBB3D = dict(K0=15, **{"K+": 15, "K-": 5}, KF=3, KS=25, KCH0=2, KCH1=2, KPOS_EVEN=5, KPOS_ODD=5, KPOS_TAIL=5, KF_EVEN=1,
             KF_ODD=1, KF_TAIL=1, KPX0=20, KPX1=8, ROUND_GE1=40)
OBB3D_HEAVY = dict(K0=15, **{"K+": 15, "K-": 5}, KF=2, KS=25, KCH0=2, KCH1=2, KPOS_EVEN=10, KPOS_ODD=5, KPX0=20, KPX1=8,
                   ROUND_GE1=40)
KNIFE_CLAIMS = {
    ("obb3d", False, False): OBB3D,
    ("obb3d", True, False): OBB3D,
    ("obb3d", False, True): OBB3D_HEAVY,
    ("obb3d", True, True): OBB3D_HEAVY,
    ("aabb3d", False, False): dict(K0=15, **{"K+": 5, "K-": 5}, KS=20, KCH0=2, KCH1=2),
    ("aabb3d", True, False): dict(K0=15, **{"K+": 5, "K-": 5}, KS=20, KCH0=2, KCH1=2),
    ("aabb2d", False, False): dict(K0=2, **{"K-": 3}, KS=8, KCH0=2, KCH1=2),
    ("aabb2d", True, False): dict(K0=1, **{"K+": 2, "K-": 2}, KS=8, KCH0=2, KCH1=2),
    ("obb2d", False, False): dict(K0=2, **{"K+": 2}, KS=8, KCH0=2, KCH1=2, KPOS_EVEN=2, KPOS_ODD=5, KPOS_TAIL=4, KPX0=20,
                                  KPX1=8),
    ("obb2d", True, False): dict(K0=2, **{"K+": 2, "K-": 2}, KS=8, KCH0=2, KCH1=2, KPOS_EVEN=3, KPOS_ODD=5, KPOS_TAIL=3,
                                 KPX0=20, KPX1=8),
}
KNIFE_KEYS = list(KNIFE_CLAIMS)


def uniform(s):
    return B.GaussianSplattingPlugin.cloud_uniform(s)


@pytest.mark.parametrize("geom,saturated,heavy", KNIFE_KEYS,
                         ids=[f"{g}-{'sat' if s else 'ord'}{'-heavy' if h else ''}" for g, s, h in KNIFE_KEYS])
def test_knife_constructions_reach_their_classes(oracle, geom, saturated, heavy):
    t0 = time.perf_counter()
    case = BC.knife_case(oracle, geom, saturated, heavy=heavy)
    cls, info = BC.pair_classes(oracle, case)
    took = time.perf_counter() - t0
    counts = {k: len(v) for k, v in cls.items()}
    if heavy:          # the frame raster2_kernel<false> gets once large_footprint_raster holds
        til = info["til"]
        assert til["n_pairs"] >= 8 * til["n_vis"]
    for k, lo in KNIFE_CLAIMS[(geom, saturated, heavy)].items():
        assert counts[k] >= lo, f"{geom} {'saturated' if saturated else 'ordinary'}: class {k} reached {counts[k]} < {lo} ({counts})"
    # the knife pairs are decided within a few ulps and their splat's colour stands out from what lies behind it
    vis = info["visible"]
    assert vis.sum() >= 0.6 * len(vis)
    tr, ranks = info["trace"], info["ranks"]
    for i in np.flatnonzero(vis):
        x, y = case.pixels[i]
        if info["probe"]["covered"][i] and tr[y, x]["rank1"] >= 0:
            c0, c1 = info["rec"][ranks[i]], info["rec"][tr[y, x]["rank1"]]
            assert min(abs(c0[k] - c1[k]) for k in ("r", "g", "b")) >= 0.1
    if saturated:
        # every knife pixel blends only clamped alphas (a few surfel-dot corners elsewhere may not)
        unc = (tr["flags"] & oracle.TRACE_UNCLAMPED) != 0
        assert not np.any(unc[case.pixels[:, 1], case.pixels[:, 0]]) and unc.mean() < 0.01
    assert took < 30, took


@pytest.mark.parametrize("geom", list(BC.GEOMETRIES))
def test_saturated_frames_are_coverage_maps(oracle, geom):
    """Every blended alpha is the clamp, and most pixels have two covering splats (so a flipped decision of either moves
    the pixel by >= 1e-4)."""
    cloud, view, s = BC.saturated_case(geom)
    tr = oracle.blend_trace(cloud, view.to_abi(), uniform(s), s.to_abi())
    assert not np.any(tr["flags"] & (oracle.TRACE_UNCLAMPED | oracle.TRACE_NEAR_STOP))
    assert (tr["n_blended"] >= 2).mean() > 0.95 and tr["n_blended"].max() == 2
    np.testing.assert_array_equal(tr["T"][tr["n_blended"] == 2], np.float32(1 - np.float32(0.999)) * np.float32(1 - np.float32(0.999)))


def replay_f32(oracle, cloud, view, s):
    """f32 replay of tile_mode from `coverage_probe` decisions: per pixel, its tile's slice in order, w = a T, c += w c,
    T *= 1 - a, stop at T < T_STOP.  -> (image rgb, T, n_blended)."""
    u = uniform(s)
    til = oracle.render_tiles(cloud, view.to_abi(), u, s.to_abi())
    rec = oracle.project(cloud, view.to_abi(), u, s.to_abi(), til["rank_to_id"])
    W, H = view.width, view.height
    tx = -(-W // 16)
    img = np.zeros((H, W, 3), np.float32)
    Tm = np.ones((H, W), np.float32)
    nb = np.zeros((H, W), np.int64)
    f = np.float32
    for y in range(H):
        for x in range(W):
            a0, a1 = til["tile_ranges"][(y // 16) * tx + x // 16]
            sl = til["tile_entries"][a0:a1]
            if len(sl) == 0:
                continue
            pr = oracle.coverage_probe(rec[sl], s.to_abi(), np.tile([[x + 0.5, y + 0.5]], (len(sl), 1)))
            T, c = f(1), np.zeros(3, np.float32)
            for j in np.flatnonzero(pr["covered"]):
                a = pr["alpha"][j]
                w = f(a * T)
                r = rec[sl[j]]
                c = (c + np.array([w * r["r"], w * r["g"], w * r["b"]], np.float32)).astype(np.float32)
                T = f(T * f(f(1) - a))
                nb[y, x] += 1
                if T < f(BC.T_STOP):
                    break
            img[y, x], Tm[y, x] = c, T
    return til, img, Tm, nb


@pytest.mark.parametrize("geom", list(BC.GEOMETRIES))
def test_probe_and_trace_reproduce_render_tiles(oracle, geom):
    """The probe's decisions and alphas, replayed in f32, give render_tiles' image bit for bit, and the trace stops
    where that replay stops (T and the blended count)."""
    cloud = B.random_gaussians_3d_seeded(1500, 3 + list(BC.GEOMETRIES).index(geom))
    gm, aabb = BC.GEOMETRIES[geom]
    s = B.CloudSettings(global_scale=0.3, gaussian_mode=gm, aabb=aabb)
    view = B.headless_view(72, 40)
    til, img, T, nb = replay_f32(oracle, cloud, view, s)
    np.testing.assert_array_equal(img, til["image"][..., :3])
    tr = oracle.blend_trace(cloud, view.to_abi(), uniform(s), s.to_abi())
    np.testing.assert_array_equal(tr["T"], T)
    np.testing.assert_array_equal(tr["n_blended"].astype(np.int64), nb)
    assert nb.max() >= 3 and (nb > 0).mean() > 0.3


def test_probe_fused_and_unfused_decisions(oracle):
    """covered_if_unfused recomputes u, v as rounded multiply + rounded add: it agrees with the fma decision away from
    the edge and differs somewhere on the knife edges built for it."""
    case = BC.knife_case(oracle, "obb3d", False)
    cls, info = BC.pair_classes(oracle, case)
    pr = info["probe"]
    far = np.abs(info["du"]) > 64
    assert np.all(pr["covered"][far] == pr["covered_if_unfused"][far])
    assert len(cls["KF"]) > 0


CPU_BOUND_CASES = [("obb3d", 8000, 0.25), ("aabb3d", 6000, 0.25), ("aabb2d", 6000, 0.12), ("obb2d", 6000, 0.2)]


@pytest.mark.parametrize("geom,n,scale", CPU_BOUND_CASES)
def test_oracle_f32_blend_within_bound_of_c64(oracle, geom, n, scale):
    """The oracle's f32 tile_mode image against the trace's float64 blend: within the per-pixel bound everywhere, and
    the bound is not vacuous: away from stop-flagged pixels it is a few 1e-6 of the pixel's largest colour (measured
    at most 2.4e-6 max|c| on these frames, up to 14 blended splats), 400x under the flat 1e-3 bar."""
    gm, aabb = BC.GEOMETRIES[geom]
    cloud = B.random_gaussians_3d_seeded(n, 21)
    s = B.CloudSettings(global_scale=scale, gaussian_mode=gm, aabb=aabb)
    view = B.headless_view(200, 120)
    u = uniform(s)
    img = oracle.render_tiles(cloud, view.to_abi(), u, s.to_abi())["image"]
    tr = oracle.blend_trace(cloud, view.to_abi(), u, s.to_abi())
    bound, ns = BC.frame_bounds(tr, aabb, "opaque")
    err = np.abs(img.astype(np.float64) - BC.expected_frame(tr, "opaque"))
    ratio = np.where(bound > 0, err / np.where(bound > 0, bound, 1), np.where(err > 0, np.inf, 0))
    assert ratio.max() <= 1.0, (ratio.max(), np.unravel_index(ratio.argmax(), ratio.shape))
    assert (tr["n_blended"] > 0).mean() > 0.5
    m = tr["max_c"].astype(np.float64)[..., None]
    assert np.all(bound[~ns][..., :3] <= 5e-6 * m[~ns])
