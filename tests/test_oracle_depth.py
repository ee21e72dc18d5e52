"""The depth-tested frame's oracle (depth_oracle/, the rule in include/bgs.h at bgs_render_depth_test), no GPU.

* d: an independent numpy f32 restatement equals the oracle's bit for bit (off-axis cameras, a rotated and scaled model
  matrix, splats with h.w small enough that pw < 1), and a splat drawn with h.w in (-1e-9, 0) has d < 0;
* with no buffer the depth oracle's walks are the oracle's own, bit for bit;
* ref_mode equals tile_mode with a depth buffer; a zero buffer changes nothing (but hides the h.w < 0 splat); a buffer
  at or above every d gives the clear frame;
* knife buffers flip a pixel's first decision exactly between d and nextafter(d, +inf)."""
import dataclasses

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
from bevy_gaussian_splatting_b200.camera import View, look_at_rh
from depth_oracle import depth_oracle as D


def uniform(s, transform=None):
    return B.GaussianSplattingPlugin.cloud_uniform(s, transform)


def np_splat_depth(pos, model, clip):
    """include/bgs.h's d in numpy f32, every step rounded in the order written (no contraction)."""
    f = np.float32
    p = pos[:, :3].astype(f)

    def mat4_point(m, x, y, z):   # m: 16 column-major
        m = np.asarray(m, f)
        return [((m[0 + r] * x + m[4 + r] * y) + m[8 + r] * z) + m[12 + r] for r in range(4)]

    pw = mat4_point(model, p[:, 0], p[:, 1], p[:, 2])
    h = mat4_point(clip, pw[0], pw[1], pw[2])
    den = h[3] + f(1e-9)
    with np.errstate(divide="ignore", invalid="ignore"):
        return (h[2] / den) / (h[3] / den)


def off_axis_view(w=200, h=150, eye=(2.5, 1.2, 6.0), target=(0.3, -0.2, 0.0), skew=0.2):
    v = B.headless_view(w, h)
    view_from_world = look_at_rh(np.array(eye, np.float32), np.array(target, np.float32), np.array([0, 1, 0], np.float32))
    proj = v.clip_from_view.copy()
    proj[0, 2] += skew           # an off-centre (asymmetric) frustum
    return View(view_from_world=view_from_world, clip_from_view=proj, world_position=np.array(eye, np.float32), width=w, height=h)


def model_matrix():
    a = 0.7
    r = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    m = np.eye(4)
    m[:3, :3] = r @ np.diag([1.3, 0.8, 1.1])
    m[:3, 3] = [0.2, -0.1, 0.3]
    return B.CloudTransform(m.astype(np.float32))


@pytest.mark.parametrize("case", ["headless", "off_axis", "off_axis_model"])
def test_splat_depth_bit_exact(case):
    cloud = B.random_gaussians_3d_seeded(3000, 3)
    view = B.headless_view(160, 120) if case == "headless" else off_axis_view()
    tr = model_matrix() if case == "off_axis_model" else None
    u = uniform(B.CloudSettings(), tr)
    pos = cloud.position_visibility.copy()
    # a few splats just in front of the camera plane: h.w small, pw = h.w / (h.w + 1e-9) < 1
    eye = np.linalg.inv(view.view_from_world.astype(np.float64))[:3, 3]
    fwd = -np.linalg.inv(view.view_from_world.astype(np.float64))[:3, 2]
    for k, t in enumerate([1e-6, 3e-7, 1e-7, 4e-8]):
        pos[k, :3] = (eye + t * fwd).astype(np.float32)
    ids = np.arange(len(pos), dtype=np.uint32)
    va = view.to_abi()
    got = D.splat_depth(pos, va, u, ids)
    want = np_splat_depth(pos, np.array(u.transform, np.float32), np.array(va.clip_from_world, np.float32))
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    if tr is None:
        h = np.array(va.clip_from_world, np.float32).reshape(4, 4).T.astype(np.float64) @ np.c_[pos[:4, :3], np.ones(4)].T
        pw = h[3] / (h[3] + 1e-9)
        assert (pw < 1.0).all()


def test_negative_w_splat_is_drawn_and_a_zero_buffer_hides_it():
    """h.w in (-1e-9, 0): the frustum test passes (x, y, z tiny), pw < 0 and d < 0, so a cleared buffer hides it."""
    view = B.headless_view(64, 48)
    va = view.to_abi()
    m = np.zeros(16, np.float32)
    m[12], m[13], m[14], m[15] = 0.0, 0.0, 2e-10, -5e-10      # h = (0, 0, 2e-10, -5e-10) for every position
    va.clip_from_world[:] = m.tolist()
    pos = np.array([[0.0, 0.0, 0.0, 1.0]], np.float32)
    d = D.splat_depth(pos, va, uniform(B.CloudSettings()), np.array([0], np.uint32))
    assert d[0] < 0.0
    from oracle import oracle as O
    assert O.keygen(pos, va, uniform(B.CloudSettings()), 32)[0] != 0xFFFFFFFF     # drawn (in the frustum)
    # rendered: every splat lands at the frame's centre; a zero buffer hides all of them, in both walks
    cloud = B.random_gaussians_3d_seeded(50, 13)
    s = B.CloudSettings(global_scale=0.5, color_space=B.GaussianColorSpace.LinRec709Display)
    u, sa = uniform(s), s.to_abi()
    zero = np.zeros((view.height, view.width), np.float32)
    clear = np.zeros((view.height, view.width, 4), np.float32)
    clear[..., 3] = 1.0
    assert not np.array_equal(D.render_tiles(cloud, va, u, sa), clear)
    assert not np.array_equal(D.render_ref(cloud, va, u, sa), clear)
    assert np.array_equal(D.render_tiles(cloud, va, u, sa, zero), clear)
    assert np.array_equal(D.render_ref(cloud, va, u, sa, zero), clear)


def small_scene(seed=0, n=600, w=96, h=80):
    cloud = B.random_gaussians_3d_seeded(n, seed)
    view = B.headless_view(w, h)
    s = B.CloudSettings(global_scale=0.6, color_space=B.GaussianColorSpace.LinRec709Display)
    return cloud, view, s


def dataclasses_asdict(s):
    return {f.name: getattr(s, f.name) for f in dataclasses.fields(s)}


GEOMS = {"obb3d": dict(), "aabb3d": dict(aabb=True), "obb2d": dict(gaussian_mode=B.GaussianMode.Gaussian2d),
         "aabb2d": dict(aabb=True, gaussian_mode=B.GaussianMode.Gaussian2d)}


@pytest.mark.parametrize("geom", list(GEOMS))
@pytest.mark.parametrize("seed", [0, 4])
def test_no_buffer_is_the_oracles_walk(oracle, geom, seed):
    """depth_oracle's walks restate the oracle's with the test added: with no buffer they are the oracle's, bit for bit,
    for every geometry (each walk's decision and blend code is the oracle's own, compiled in)."""
    cloud, view, s = small_scene(seed)
    s = B.CloudSettings(**{**dataclasses_asdict(s), **GEOMS[geom]})
    va, u, sa = view.to_abi(), uniform(s), s.to_abi()
    til = oracle.render_tiles(cloud, va, u, sa)
    assert np.array_equal(D.render_tiles(cloud, va, u, sa).view(np.uint32), til["image"].view(np.uint32))
    assert np.array_equal(D.render_ref(cloud, va, u, sa).view(np.uint32), oracle.render_ref(cloud, va, u, sa).view(np.uint32))
    assert np.array_equal(D.blend_trace(cloud, va, u, sa).view(np.uint8), oracle.blend_trace(cloud, va, u, sa).view(np.uint8))


def plane_buffer(view, cloud, u, frac=0.5):
    """Reverse-Z occluder: the left `frac` of the frame at the median splat depth, the rest cleared."""
    d = D.splat_depth(cloud.position_visibility, view.to_abi(), u, np.arange(len(cloud), dtype=np.uint32))
    z = np.zeros((view.height, view.width), np.float32)
    z[:, : int(frac * view.width)] = np.median(d[np.isfinite(d) & (d > 0)])
    return z


def test_ref_mode_equals_tile_mode_with_a_buffer(oracle):
    cloud, view, s = small_scene(1)
    va, u, sa = view.to_abi(), uniform(s), s.to_abi()
    z = plane_buffer(view, cloud, u)
    ref, til = D.render_ref(cloud, va, u, sa, z), D.render_tiles(cloud, va, u, sa, z)
    assert float(np.abs(ref - til).max()) <= 1e-3
    # the occluder changed the covered half and only it
    plain = D.render_tiles(cloud, va, u, sa)
    half = view.width // 2
    assert not np.array_equal(til[:, :half], plain[:, :half])
    assert np.array_equal(til[:, half:], plain[:, half:])


def test_zero_buffer_changes_nothing_and_a_far_buffer_hides_everything(oracle):
    cloud, view, s = small_scene(2)
    va, u, sa = view.to_abi(), uniform(s), s.to_abi()
    zero = np.zeros((view.height, view.width), np.float32)
    assert np.array_equal(D.render_tiles(cloud, va, u, sa, zero).view(np.uint32), D.render_tiles(cloud, va, u, sa).view(np.uint32))
    assert np.array_equal(D.render_ref(cloud, va, u, sa, -zero).view(np.uint32), D.render_ref(cloud, va, u, sa).view(np.uint32))
    d = D.splat_depth(cloud.position_visibility, va, u, np.arange(len(cloud), dtype=np.uint32))
    for far in (np.float32(d[np.isfinite(d)].max()), np.float32(np.inf), np.float32(np.nan)):
        img = D.render_tiles(cloud, va, u, sa, np.full((view.height, view.width), far, np.float32))
        hidden = D.render_tiles(cloud, va, u, sa, np.full((view.height, view.width), np.nextafter(far, np.float32(np.inf)), np.float32))
        clear = np.zeros_like(img)
        clear[..., 3] = 1.0
        assert np.array_equal(hidden, clear)
        if not np.isfinite(far):
            assert np.array_equal(img, clear)


def test_knife_buffers_flip_the_first_decision_between_d_and_nextafter(oracle):
    cloud, view, s = small_scene(3)
    va, u, sa = view.to_abi(), uniform(s), s.to_abi()
    tr = D.blend_trace(cloud, va, u, sa)
    til = oracle.render_tiles(cloud, va, u, sa, want_image=False)
    d_rank = D.splat_depth(cloud.position_visibility, va, u, til["rank_to_id"])
    ys, xs = np.nonzero(tr["rank0"] >= 0)
    pick = np.random.default_rng(0).choice(len(ys), 200, replace=False)
    for k in pick[:40]:
        y, x = ys[k], xs[k]
        r0 = tr["rank0"][y, x]
        at = np.zeros((view.height, view.width), np.float32)
        at[y, x] = d_rank[r0]
        above = at.copy()
        above[y, x] = np.nextafter(d_rank[r0], np.float32(np.inf))
        assert D.blend_trace(cloud, va, u, sa, at)["rank0"][y, x] == r0
        assert D.blend_trace(cloud, va, u, sa, above)["rank0"][y, x] != r0
    # the probe makes the same decision pair by pair
    rec = oracle.project(cloud, va, u, sa, til["rank_to_id"][tr["rank0"][ys[pick], xs[pick]]])
    xy = np.stack([xs[pick] + 0.5, ys[pick] + 0.5], 1)
    dd = d_rank[tr["rank0"][ys[pick], xs[pick]]]
    assert D.coverage_probe(rec, sa, xy, dd, dd)["covered"].all()
    assert not D.coverage_probe(rec, sa, xy, dd, np.nextafter(dd, np.float32(np.inf)))["covered"].any()
