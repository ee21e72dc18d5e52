"""bgs_render_4d's rule on the CPU: temporal_oracle/ against tests/temporal_cases.py's numpy restatement, bit for bit,
on the inputs that sit on the rule's decisions; the .ply4d reader and writer; playback_update against settings.rs."""
import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import project_cases as PC
import temporal_cases as TC
from temporal_oracle import temporal_oracle as T

f32 = np.float32


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def test_exp_and_cos_series_agree():
    rng = np.random.default_rng(0)
    x = np.concatenate([-rng.random(500, np.float32) * 120, [0.0, -0.0, -1e-30, -103.9, -104.0, -110.0, -110.1, 88.9, 89.1,
                                                             np.nan, -np.inf, np.inf]]).astype(np.float32)
    assert np.array_equal(bits(T.exp(x)), bits(TC.det_exp(x)))
    fin = np.isfinite(x) & (x > -80) & (x < 80)
    assert np.allclose(T.exp(x)[fin], np.exp(x[fin].astype(np.float64)), rtol=2 ** -23, atol=0)
    c = np.concatenate([(rng.random(500, np.float32) - 0.5) * 200, [0.0, -0.0, np.pi, 2 * np.pi, 1e6, np.nan, np.inf]]).astype(np.float32)
    assert np.array_equal(bits(T.cos(c)), bits(TC.det_cos(c)), equal_nan=False) or \
        np.array_equal(np.isnan(T.cos(c)), np.isnan(TC.det_cos(c)))
    ok = ~np.isnan(c)
    assert np.array_equal(bits(T.cos(c)[ok & np.isfinite(c)]), bits(TC.det_cos(c)[ok & np.isfinite(c)]))
    small = np.abs(c) < 1000
    assert np.allclose(T.cos(c)[small], np.cos(c[small].astype(np.float64)), atol=2 ** -24 * 1.5, rtol=0)


def _agree(rot8, so, tt, gs, t):
    o = T.condition(rot8, so, tt, gs, t)
    cov6, dm, marg, mask = TC.condition(rot8, so, tt, gs, t)
    assert np.array_equal(o["mask"], mask)
    assert np.array_equal(bits(o["marginal"]), bits(marg))
    assert np.array_equal(bits(o["cov6"]), bits(cov6))
    assert np.array_equal(bits(o["delta_mean"]), bits(dm))
    return o


def _cloud(n, seed):
    c = B.random_gaussians_4d_seeded(n, seed)
    return c.isotropic_rotations, c.scale_opacity, c.timestamp_timescale


def test_conditioning_random_and_unnormalised():
    rot8, so, tt = _cloud(3000, 1)
    assert np.abs(np.linalg.norm(rot8[:, :4], axis=1) - 1).max() > 0.1   # unnormalised quaternions, as generated
    for t in (0.0, 0.3, 0.77, 1.5):
        o = _agree(rot8, so, tt, 1.0, t)
        assert 0 < o["mask"].sum() < len(rot8)
    _agree(rot8 * f32(3.0), so, tt, 0.5, 0.4)


def test_marginal_ulp_walk_across_threshold():
    """Timescales walked ulp by ulp so that marginal_t crosses 0.05: the draw decision is bit-exact."""
    rot8 = np.tile(np.array([1, 0, 0, 0, 1, 0, 0, 0], np.float32), (1, 1))
    # identity rotations: cov_t = timescale^2; marginal = exp(-0.5 dt^2 / st^2) = 0.05 at st = dt / sqrt(2 ln 20)
    dt = f32(0.5)
    st0 = f32(float(dt) / np.sqrt(2 * np.log(20.0)))
    st = PC.ulp_walk(np.array([st0], np.float32), range(-64, 65)).ravel()
    n = len(st)
    rot8 = np.tile(rot8, (n, 1))
    so = np.tile(np.array([0.3, 0.2, 0.1, 0.5], np.float32), (n, 1))
    tt = np.stack([np.zeros(n, np.float32), st, np.zeros(n, np.float32), np.zeros(n, np.float32)], 1)
    o = _agree(rot8, so, tt, 1.0, dt)
    assert 0 < o["mask"].sum() < n   # the walk straddles the threshold


def test_conditioning_edges():
    n = 6
    rot8 = np.tile(np.array([1, 0, 0, 0, 1, 0, 0, 0], np.float32), (n, 1))
    so = np.tile(np.array([0.3, 0.2, 0.1, 0.5], np.float32), (n, 1))
    tt = np.array([[0.5, 0.0, 0, 0],      # cov_t = 0, dt = 0: NaN, not drawn
                   [0.2, 0.0, 0, 0],      # cov_t = 0, dt != 0: exp(-inf) = 0
                   [0.5, -0.7, 0, 0],     # negative timescale
                   [0.5, 0.3, 0, 0],      # dt = 0
                   [np.inf, 0.3, 0, 0],   # non-finite timestamp
                   [0.4, 1e-20, 0, 0]], np.float32)
    o = _agree(rot8, so, tt, 1.0, 0.5)
    assert list(o["mask"]) == [False, False, True, True, False, False]
    # a coupled rotation pair: the time axis mixes with space, delta_mean != 0
    q = np.array([[0.9, 0.3, -0.2, 0.1, 0.8, -0.4, 0.3, 0.2]], np.float32)
    o = _agree(q, so[:1], np.array([[0.3, 0.5, 0, 0]], np.float32), 1.3, 0.45)
    assert o["mask"][0] and np.abs(o["delta_mean"]).max() > 0


def test_velocity_cases():
    """v = 0 (no coupling), scaled either side of 1e-2, and a future mask that fails: the conditionings at t and
    t + 1e-3 agree bit for bit, and so does what Velocity makes of them."""
    rot8, so, tt, t = TC.fast_arrays()
    o = _agree(rot8, so, tt, 1.0, t)
    fut = _agree(rot8, so, tt, 1.0, f32(t) + f32(1e-3))
    assert (o["mask"] & ~fut["mask"]).any()
    rgb, zero = TC.velocity(rot8, so, tt, 1.0, t)
    v = np.linalg.norm((np.where(fut["mask"][:, None], fut["delta_mean"], 0) - o["delta_mean"]) / 1e-3, axis=1)
    assert ((v > 1.0) & (v < 1.01)).any() and ((v >= 1.01) & (v < 1.02)).any()
    assert zero.any() and (~zero).any()
    # identity rotations, unit scales: no coupling at all, v = 0 exactly
    ident = np.tile(np.array([1, 0, 0, 0, 1, 0, 0, 0], np.float32), (4, 1))
    _, z0 = TC.velocity(ident, np.ones((4, 4), np.float32), np.tile(np.array([0.5, 0.5, 0, 0], np.float32), (4, 1)), 1.0, 0.5)
    assert z0.all()


def _frame_case(mode, seed=0, t=0.5, draw=B.DrawMode.All, aabb=False):
    c = TC.scene_4d(600, seed, selected=True)
    v = B.headless_view(96, 64)
    s = B.CloudSettings(gaussian_mode=B.GaussianMode.Gaussian4d, rasterize_mode=mode, time=t, draw_mode=draw, aabb=aabb)
    u = B.GaussianSplattingPlugin.cloud_uniform(s, aabb=c.compute_aabb())
    return c, v, s, u


@pytest.mark.parametrize("t", [0.1, 0.5, 0.9])
def test_frame_records_follow_the_rule(t):
    """The oracle's Velocity colours and draw decisions equal the numpy restatement's."""
    c, v, s, u = _frame_case(B.RasterizeMode.Velocity, t=t)
    f = T.frame(c, v.to_abi(), u, s.to_abi(), 0.0, 1.0, want_image=False)
    ids = f["rank_to_id"]
    rec = f["records"]
    bb = rec[:, 6:8].view(np.uint32)
    drawn = ((bb[:, 0] & 0xFFFF) <= (bb[:, 0] >> 16)) & ((bb[:, 1] & 0xFFFF) <= (bb[:, 1] >> 16))
    rgb, zero = TC.velocity(c.isotropic_rotations[ids], c.scale_opacity[ids], c.timestamp_timescale[ids], 1.0, t)
    _, _, _, mask = TC.condition(c.isotropic_rotations[ids], c.scale_opacity[ids], c.timestamp_timescale[ids], 1.0, t)
    assert not (drawn & ~mask).any()
    assert drawn.sum() > 10
    assert np.array_equal(bits(rec[drawn, 8:11]), bits(rgb[drawn]))
    assert np.array_equal(rec[drawn, 11] == 0, zero[drawn])


@pytest.mark.parametrize("term", [0, 1, 2])
def test_each_time_term_alone(term):
    """One coefficient set at a time (SH degree 0 of section `term`): colour = 0.5 + C0 * sh * cos(2 pi k theta)."""
    c, v, s, u = _frame_case(B.RasterizeMode.Color, seed=2, t=0.3)
    s.color_space = B.GaussianColorSpace.LinRec709Display
    u = B.GaussianSplattingPlugin.cloud_uniform(s, aabb=c.compute_aabb())
    sh = np.zeros_like(c.spherindrical_harmonic)
    sh[:, 48 * term:48 * term + 3] = f32(0.7)
    c = B.PlanarGaussian4d(c.position_visibility, sh, c.isotropic_rotations, c.scale_opacity, c.timestamp_timescale)
    f = T.frame(c, v.to_abi(), u, s.to_abi(), 0.0, 2.0, want_image=False)
    rec, ids = f["records"], f["rank_to_id"]
    bb = rec[:, 6:8].view(np.uint32)
    drawn = ((bb[:, 0] & 0xFFFF) <= (bb[:, 0] >> 16))
    dt = (f32(0.3) - c.timestamp_timescale[ids, 0]).astype(np.float32)
    theta = (dt / f32(2.0)).astype(np.float32)
    k = [None, f32(2 * np.float32(np.pi)), f32(4 * np.float32(np.pi))][term]
    factor = np.ones_like(theta) if term == 0 else TC.det_cos((k * theta).astype(np.float32))
    want = 0.5 + 0.28209479177387814 * 0.7 * factor.astype(np.float64)
    assert drawn.sum() > 10
    assert np.abs(rec[drawn, 8] - want[drawn]).max() < 1e-6


def test_negative_duration_and_selected_mode():
    c, v, s, u = _frame_case(B.RasterizeMode.Color, seed=4, draw=B.DrawMode.Selected)
    a = T.frame(c, v.to_abi(), u, s.to_abi(), 1.0, 0.0, want_image=False)
    b = T.frame(c, v.to_abi(), u, s.to_abi(), 0.0, 1.0, want_image=False)
    bb = a["records"][:, 6:8].view(np.uint32)
    drawn = (bb[:, 0] & 0xFFFF) <= (bb[:, 0] >> 16)
    assert not (drawn & (c.position_visibility[a["rank_to_id"], 3] < 0.5)).any()
    # cos is even: a negative duration gives the same colours
    assert np.array_equal(bits(a["records"]), bits(b["records"]))


def test_ply4d_round_trip_normalisation_padding(tmp_path):
    c = B.random_gaussians_4d_seeded(45, 7)
    p = tmp_path / "c.ply4d"
    B.write_ply_4d(p, c)
    r = B.load_cloud(p)
    assert len(r) == 64   # padded to a multiple of 32
    assert np.array_equal(r.position_visibility[:45], c.position_visibility)
    assert np.array_equal(r.spherindrical_harmonic[:45], c.spherindrical_harmonic)
    assert np.array_equal(r.scale_opacity[:45], c.scale_opacity)
    assert np.array_equal(r.timestamp_timescale[:45, :2], c.timestamp_timescale[:, :2])
    for lo in (0, 4):
        q = c.isotropic_rotations[:, lo:lo + 4]
        n = np.sqrt(np.sum(q * q, axis=1, dtype=np.float32), dtype=np.float32)
        assert np.array_equal(r.isotropic_rotations[:45, lo:lo + 4], (q / n[:, None]).astype(np.float32))
    assert np.array_equal(r.position_visibility[45:, 3], np.ones(19, np.float32))
    assert not r.spherindrical_harmonic[45:].any()
    c2 = B.random_gaussians_4d_seeded(64, 1)
    B.write_ply_4d(p, c2)
    assert len(B.load_cloud(p)) == 96   # a full 32 when n is already a multiple of 32, as ply.rs pads


def test_ply4d_missing_property(tmp_path):
    c = B.random_gaussians_4d_seeded(3, 0)
    p = tmp_path / "c.ply4d"
    B.write_ply_4d(p, c)
    data = p.read_bytes().replace(b"property float rot_r_w\n", b"property float rot_r_q\n")
    with pytest.raises(ValueError):
        B.parse_ply_4d(data)


def test_playback_update_modes():
    S = B.CloudSettings
    s = S(playback_mode=B.PlaybackMode.Still, time=0.3)
    B.playback_update(s, 0.1, 5.0)
    assert s.time == f32(0.3)
    s = S(playback_mode=B.PlaybackMode.Loop, time=0.95, time_scale=2.0)
    B.playback_update(s, 0.01, 5.0)
    assert s.time == f32(f32(0.95) + f32(f32(0.01) * f32(2.0)))
    B.playback_update(s, 0.1, 5.0)
    assert s.time == 0.0   # past time_stop: wrapped to time_start
    s = S(playback_mode=B.PlaybackMode.Once, time=0.95)
    B.playback_update(s, 0.1, 5.0)
    assert s.time == f32(f32(0.95) + f32(0.1))   # Once is not clamped
    before = s.time
    B.playback_update(s, 0.1, 5.0)
    assert s.time == before   # time >= time_stop: Once stops
    s = S(playback_mode=B.PlaybackMode.Sin, time_start=1.0, time_stop=3.0, time_scale=0.25)
    B.playback_update(s, 0.1, 1.0)
    y = np.sin(f32(f32(f32(0.25) * f32(2.0)) * f32(np.pi)), dtype=np.float32)
    assert s.time == f32(f32(1.0) + f32(f32(f32(2.0) * f32(y + f32(1.0))) / f32(2.0)))
    s = S(playback_mode=B.PlaybackMode.Loop, time=0.5, time_scale=0.0)
    B.playback_update(s, 0.1, 1.0)
    assert s.time == 0.5
