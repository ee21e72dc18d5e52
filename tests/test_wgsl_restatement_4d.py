"""temporal_oracle/ against the INDEPENDENT float64 restatement of the reference's Gaussian4d rule (tests/wgsl_emu_4d.py).

CPU only.  The oracle and the kernel were written from one reading of gaussian_4d.wgsl and
spherindrical_harmonics.wgsl; the emulator is a second one.  Off-axis camera, a rotated, non-uniformly scaled and
translated model matrix, inputs from tests/temporal_wgsl_cases.py that reach each part of the rule.

Decisions (the base and moved frustum tests, the time mask, Velocity's cut, the integer bbox) must be equal; the only
exceptions are inputs whose float64 margin lies inside the f32 error bound of the quantity decided, and their count is
asserted small.  Values are held to the running error bounds of temporal_wgsl_cases (E: multiples of u = 2^-24 of the
magnitudes of the terms that produce them, derived in that module's docstring)."""
import math

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import temporal_wgsl_cases as TW
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import CloudTransform, GaussianSplattingPlugin
from oracle import oracle as O
from temporal_oracle import temporal_oracle as T
from wgsl_emu import Vec
from wgsl_emu_4d import render_reference_semantics_4d

f32 = np.float32
RM = B.RasterizeMode
W, H = 160, 112
WINDOW = (0.0, 1.0)


def extras_for(view):
    ex = abi.bgs_render_extras(num_classes=3)
    prev = B.perspective_view((2.3, 1.7, 4.6), (0.1, 0.0, -0.2), view.width, view.height, up=(0.15, 1.0, -0.05))
    ex.previous_clip_from_world[:] = prev.to_abi().clip_from_world[:]
    ex.delta_time = 1.0 / 30.0
    return ex


def case(mode, aabb=False, draw=B.DrawMode.All, cs=0, seed=0, n=256, window=WINDOW, w=W, h=H):
    cloud = TW.edge_cloud(n, seed)
    view = TW.off_axis_view(w, h)
    s = B.CloudSettings(gaussian_mode=B.GaussianMode.Gaussian4d, rasterize_mode=mode, time=0.5, aabb=aabb, draw_mode=draw,
                        color_space=B.GaussianColorSpace(cs), num_classes=3, global_scale=1.3, global_opacity=0.9,
                        time_start=window[0], time_stop=window[1])
    u = GaussianSplattingPlugin.cloud_uniform(s, CloudTransform(TW.model_matrix()), cloud.compute_aabb())
    return cloud, view, s, u


def sorted_ids(cloud, view, u):
    keys = O.keygen(cloud.position_visibility, view.to_abi(), u, 32)
    return O.radix_sort(keys, 32)[1]


CASES = [(m, aabb, draw, cs) for m in [RM.Color, RM.Depth, RM.Position, RM.Classification, RM.OpticalFlow, RM.Velocity]
         for aabb in (False, True) for draw, cs in ((B.DrawMode.All, 0), (B.DrawMode.Selected, 1), (B.DrawMode.HighlightSelected, 0))]


@pytest.mark.parametrize("mode,aabb,draw,cs", CASES, ids=[f"{m.name}-{'aabb' if a else 'obb'}-{d.name}-cs{c}" for m, a, d, c in CASES])
def test_records_match_wgsl_restatement(mode, aabb, draw, cs):
    cloud, view, s, u = case(mode, aabb, draw, cs)
    ex = extras_for(view)
    f = T.frame(cloud, view.to_abi(), u, s.to_abi(), *WINDOW, extras=ex, want_image=False)
    ids = f["rank_to_id"]
    compared, undecided, expected = TW.check_records(f["records"], ids, cloud, view, u, s, WINDOW, sorted_ids(cloud, view, u), ex)
    assert compared >= 60 and compared + undecided == len(ids), (compared, undecided, len(ids))
    assert undecided <= 2 * expected + 4, (undecided, expected)


def test_conditioning_matches_wgsl_restatement():
    """cov3d, delta_mean, marginal_t and the mask of every edge row at several times, unnormalised rotations, a
    negative timescale, dt = 0, marginal_t a few ulps from 0.05 and tiny cov_t."""
    cloud = TW.edge_cloud(512, 3)
    _, view, s, u = case(RM.Color)
    sh4 = TW.shader_for(view, u, s, WINDOW)
    near = 0
    for t in (0.5, 0.31, 0.77):
        o = T.condition(cloud.isotropic_rotations, cloud.scale_opacity, cloud.timestamp_timescale, 1.3, t)
        for i in range(len(cloud)):
            q8 = [float(x) for x in cloud.isotropic_rotations[i]]
            so = [float(x) for x in cloud.scale_opacity[i]]
            tt = [float(x) for x in cloud.timestamp_timescale[i]]
            g = TW.condition(float(f32(1.3)), q8, so, tt, float(f32(t)))
            em = sh4.conditional_cov3d(Vec(*q8[:4]), Vec(*q8[4:]), Vec(*so[:3]), tt[0], tt[1], float(f32(t)))
            assert abs(em["marginal_t"] - g["marginal"].v) <= 1e-12 * max(1.0, em["marginal_t"])
            if abs(em["marginal_t"] - 0.05) <= g["marginal"].bound:
                near += i % 8 != 2     # rows 2 mod 8 are built there
                continue
            assert bool(o["mask"][i]) == em["mask"], (i, t, em["marginal_t"])
            assert abs(o["marginal"][i] - em["marginal_t"]) <= g["marginal"].bound
            if not em["mask"]:
                continue
            for k in range(6):
                assert abs(o["cov6"][i, k] - em["cov3d"][k]) <= g["c3"][k].bound, (i, k)
            for k in range(3):
                assert abs(o["delta_mean"][i, k] - em["delta_mean"][k]) <= g["dm"][k].bound, (i, k)
    assert near <= 3, near
    rows2 = np.arange(len(cloud)) % 8 == 2
    o = T.condition(cloud.isotropic_rotations, cloud.scale_opacity, cloud.timestamp_timescale, 1.3, 0.5)
    assert o["mask"][rows2].any() and (~o["mask"][rows2]).any()      # the ulp walk straddles 0.05


@pytest.mark.parametrize("block", [0, 1, 2])
def test_each_coefficient_block_alone(block):
    """Rows 4, 5, 6 mod 8 carry one block each: the colour is 0.5 + the spatial sum, + t1 s1, or + t2 s2."""
    cloud, view, s, u = case(RM.Color, cs=1, n=512, seed=4)
    keep = np.arange(len(cloud)) % 8 == 4 + block
    cloud = cloud.subset(np.flatnonzero(keep))
    f = T.frame(cloud, view.to_abi(), u, s.to_abi(), *WINDOW, want_image=False)
    compared, undecided, expected = TW.check_records(f["records"], f["rank_to_id"], cloud, view, u, s, WINDOW, sorted_ids(cloud, view, u))
    assert compared >= 20 and undecided <= 2 * expected + 4
    assert not cloud.spherindrical_harmonic[:, [j for j in range(144) if j // 48 != block]].any()


@pytest.mark.parametrize("window", [(0.0, 1.0), (1.0, 0.0), (0.25, 0.75), (-3.0, 5.0)])
def test_theta_values_and_negative_duration(window):
    """theta = 0, +-1/4, +-1/2, 1 and large, for a positive and a negative duration (cos is even: the colour must not
    change sign with the duration, and the emulator says which value it takes)."""
    d = window[1] - window[0]
    thetas = [0.0, 0.25, -0.25, 0.5, -0.5, 1.0, 3.75, -12.5, 300.25]
    cloud = TW.theta_cloud([t * d for t in thetas] * 4, seed=5)
    view = TW.off_axis_view(W, H)
    s = B.CloudSettings(gaussian_mode=B.GaussianMode.Gaussian4d, rasterize_mode=RM.Color, time=0.5,
                        color_space=B.GaussianColorSpace.LinRec709Display, time_start=window[0], time_stop=window[1])
    u = GaussianSplattingPlugin.cloud_uniform(s, CloudTransform(TW.model_matrix()), cloud.compute_aabb())
    f = T.frame(cloud, view.to_abi(), u, s.to_abi(), *window, want_image=False)
    compared, undecided, expected = TW.check_records(f["records"], f["rank_to_id"], cloud, view, u, s, window, sorted_ids(cloud, view, u))
    assert compared >= 30 and undecided <= 2 * expected + 2


@pytest.mark.parametrize("mode,aabb", [(RM.Color, False), (RM.Color, True), (RM.Velocity, False), (RM.Position, True)])
def test_frame_matches_wgsl_walk(mode, aabb):
    """Small frames (63 splats, without the rows built on the time threshold): the oracle's tile walk against the emulator's quad walk, every pixel within the
    per-pixel bound temporal_wgsl_cases.check_frame derives from the records' bounds, the undecided pixels within twice
    the count those bounds predict, plus four (for an expected count below one a Poisson count still reaches 2 or 3
    a few times in a hundred; 5 or more has probability below 0.4 %).  The walk's order comes from the keys, not from
    the oracle's frame.  In Velocity mode every splat has opacity 0 (delta_mean is 0, see temporal_wgsl_cases), so
    that frame checks only that nothing is drawn."""
    cloud, view, s, u = case(mode, aabb, n=72, seed=7, w=96, h=64)
    cloud = cloud.subset(np.flatnonzero(np.arange(72) % 8 != 2))     # 63 splats: not the rows built on the time threshold
    s.color_space = B.GaussianColorSpace.LinRec709Display
    u = GaussianSplattingPlugin.cloud_uniform(s, CloudTransform(TW.model_matrix()), cloud.compute_aabb())
    f = T.frame(cloud, view.to_abi(), u, s.to_abi(), *WINDOW)
    bounds = {}
    order = TW.frame_order(cloud, view, u)
    _, rec_undecided, rec_expected = TW.check_records(f["records"], f["rank_to_id"], cloud, view, u, s, WINDOW, None,
                                                      bounds=bounds)
    assert rec_undecided <= 2 * rec_expected + 4
    sh4 = TW.shader_for(view, u, s, WINDOW)
    compared, undecided, expected, want = TW.check_frame(f["image"], cloud, sh4, order, f["records"], f["rank_to_id"], bounds)
    if mode != RM.Velocity:
        assert (np.nan_to_num(want).max(axis=2) > 0.02).sum() >= 100
    # the front-to-back walk is the emulator's back-to-front one wherever no pixel stops (none does in these frames)
    ref = render_reference_semantics_4d(sh4, cloud, order, view.width, view.height)
    ok = np.isfinite(want)
    assert np.abs(ref[..., :3][ok] - want[ok]).max() <= 1e-12
    assert undecided <= 2 * expected + 4, (undecided, expected)
    assert compared >= 0.9 * view.width * view.height


def test_det_cos_accuracy():
    """det_cos against math.cos of the same f32 argument, over every decade of the reachable range: within
    det_cos_bound (|x| 1.5005e-16 + 2^-25: the one f64 rounding of k 2pi and the f64 constant's own error, then the
    f32 rounding).  Up to |x| = 1e8 that is about half an ulp; at 1e10 1.5e-6; at 1e12 1.5e-4; at 1e15 0.15.  The
    decades run to 1e16, where the bound reaches 1.5; above that the result is not bounded at all."""
    rng = np.random.default_rng(11)
    worst = {}
    for dec in range(-3, 16):
        x = (10.0 ** (dec + rng.random(4000))) * rng.choice([-1.0, 1.0], 4000)
        x = x.astype(np.float32)
        got = T.cos(x).astype(np.float64)
        want = np.cos(x.astype(np.float64))
        err = np.abs(got - want)
        bound = np.array([TW.det_cos_bound(float(v)) for v in x])
        assert (err <= bound).all(), (dec, float(err.max()), float(x[np.argmax(err - bound)]))
        worst[dec] = float(err.max())
    # worst[d]: arguments in [1e(d), 1e(d+1))
    assert worst[7] < 5e-8 and worst[8] < 2e-7 and 1e-7 < worst[9] < 2e-6 and 1e-5 < worst[11] < 2e-4
    # past |x| ~ 1e16 the reduced argument leaves the series' range: the result is unbounded, as include/bgs.h states
    big = T.cos(np.array([1e18, 1e30], np.float32))
    assert big[0] > 1e30 and np.isposinf(big[1]), big
