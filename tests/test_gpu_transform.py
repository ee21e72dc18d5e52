"""bgs_cloud_transform and bgs_cloud_bounds on the GPU: the bake against the CPU oracle (transform_oracle/) in every layout,
SH degree, matrix class and mode, at 200 000 gaussians and at 6 M f16 / 2 M f32; render equivalence of a baked cloud
with the original drawn under uniform.transform = M; both device copies written; the queued ordering across contexts
with no host synchronisation in between; the bounds against numpy; the refusals; and launch counts of a context that
never transforms."""
import ctypes as C
import functools

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import transform_cases as TC
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.gaussian import compute_aabb
from particle_oracle import particle_oracle as PO
from test_oracle_interpolate import f32_same, half_words_same
from transform_oracle import transform_oracle as TO

pytestmark = pytest.mark.gpu

F = np.float32
N = 200_000
# SH lanes: |got - want| <= SH_REL * sum_j |E_ij c_j| (+ one f16 ulp of the result in the f16 layouts).  The two sides
# evaluate the same f32 sum in the same order; they differ only where an entry of E rounds to a neighbouring f32 (the
# library and the oracle build D_l from different direction sets), which moves each product by <= 2^-24 of itself and
# each of the <= 7 roundings of the sum by at most as much: 8 * 2^-24 = 2^-21.
SH_REL = 2.0 ** -21


@pytest.fixture(scope="module")
def plugin():
    p = B.GaussianSplattingPlugin(0)
    yield p
    p.destroy()


def _ptr(a):
    return np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)


def upload(plugin, layout, degree, planes):
    """A resident cloud holding exactly these upload planes at this SH degree."""
    planes = [np.ascontiguousarray(p) for p in planes]
    n, h, lib = len(planes[0]), C.c_void_p(), plugin._lib
    up = {"f32": lib.bgs_cloud_upload_f32_sh, "f16": lib.bgs_cloud_upload_f16_sh, "cov": lib.bgs_cloud_upload_f16_cov_sh}[layout]
    plugin._check(up(plugin._ctx, n, degree, *(_ptr(p) for p in planes), C.byref(h)))
    return B.PlanarGaussian3dHandle._adopt(plugin, h, n, layout != "f32", layout == "cov")


def _halves(words):
    w = np.asarray(words, np.uint32)
    lo = (w & 0xFFFF).astype(np.uint16).view(np.float16).astype(F)
    hi = (w >> 16).astype(np.uint16).view(np.float16).astype(F)
    return np.stack([lo, hi], -1).reshape(len(w), -1)


def _ulp16(v):
    a = np.abs(v.astype(np.float64))
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return 2.0 ** (e - 10)


def assert_transformed(layout, degree, got, want, bound, orig, hit, what):
    """Every plane but SH bit for bit (NaN equal to NaN); SH lanes within the bound; untouched gaussians byte for
    byte the upload's."""
    names = ("pos_vis", "sh", "rot", "scale_opacity") if layout == "f32" else ("pos_vis", "sh_packed", "second")
    for k, (name, g, w) in enumerate(zip(names, got, want)):
        if k == 1:
            continue
        same = f32_same(g, w) if (layout == "f32" or k == 0) else half_words_same(g, w)
        assert same, f"{what}: {layout} {name} differs"
    for g, o in zip(got, orig):
        assert np.array_equal(np.asarray(g)[~hit].view(np.uint32), np.asarray(o)[~hit].view(np.uint32)), f"{what}: untouched"
    if layout == "f32":
        g, w, tol = got[1], want[1], SH_REL * bound
    else:
        g, w = _halves(got[1]), _halves(want[1])
        tol = SH_REL * bound + np.where(bound > 0, _ulp16(w), 0.0)
    with np.errstate(invalid="ignore"):
        ok = (np.abs(g.astype(np.float64) - w) <= tol) | (np.isnan(g) & np.isnan(w)) | (g.view(np.uint32) == w.view(np.uint32))
    if not ok.all():
        bad = np.argwhere(~ok)[:4]
        raise AssertionError(f"{what}: {layout} SH lanes {bad.tolist()} got {[g[tuple(i)] for i in bad]} "
                             f"want {[w[tuple(i)] for i in bad]} bound {[tol[tuple(i)] for i in bad]}")


@functools.lru_cache(maxsize=None)
def base_planes(layout, degree, unit=True):
    return TC.planes_of(TC.cloud(N, degree, 11 + degree, unit=unit), layout)


CLASSES = [(layout, degree, name) for layout in TC.LAYOUTS for degree in TC.DEGREES for name in TC.ACCEPTED
           if degree == 3 or name in ("general", "turn_y", "identity")]


# ---- 1. the bake against the oracle ---------------------------------------------------------------------------------
@pytest.mark.parametrize("sel", [False, True], ids=["all", "selected"])
@pytest.mark.parametrize("layout,degree,name", CLASSES, ids=[f"{l}-d{d}-{n}" for l, d, n in CLASSES])
def test_transform_matches_oracle(plugin, layout, degree, name, sel):
    planes = base_planes(layout, degree, unit=(name != "general" or layout != "f32"))
    M = TC.ACCEPTED[name]
    h = upload(plugin, layout, degree, planes)
    try:
        plugin.transform(h, M, selected=sel)
        got = plugin.download_planes(h)
        want, bound = TO.transform(layout, degree, planes, M, selected=sel)
        hit = TC.selected(planes[0][:, 3]) if sel else np.ones(N, bool)
        assert 0 < hit.sum() < N or not sel
        assert_transformed(layout, degree, got, want, bound, planes, hit, f"{name} sel={sel}")
        assert plugin.sync()
    finally:
        h.destroy()


@pytest.mark.parametrize("layout,n", [("f16", 6_000_000), ("f32", 2_000_000)])
def test_transform_matches_oracle_at_scale(plugin, layout, n):
    c = B.random_gaussians_3d_seeded(n, 1)
    c.position_visibility[:, 3] = (np.random.default_rng(1).random(n) < 0.5).astype(F)
    planes = TC.planes_of(c, layout)
    h = upload(plugin, layout, 3, planes)
    try:
        state = planes
        for sel in (False, True):
            plugin.transform(h, TC.ACCEPTED["general"], selected=sel)
            want, bound = TO.transform(layout, 3, state, TC.ACCEPTED["general"], selected=sel)
            got = plugin.download_planes(h)
            hit = TC.selected(state[0][:, 3]) if sel else np.ones(n, bool)
            assert_transformed(layout, 3, got, want, bound, state, hit, f"{layout} {n} sel={sel}")
            state = got
    finally:
        h.destroy()


# ---- 2. render equivalence: the baked cloud under identity == the original under uniform.transform = M ------------
RENDER_MODES = [("3dgs_obb", {}), ("3dgs_aabb", dict(aabb=True)), ("2dgs", dict(gaussian_mode=B.GaussianMode.Gaussian2d))]


def _render(plugin, h, settings, view, transform=None):
    img = plugin.render_view(h, settings, view, transform=transform, fmt="rgba32f").copy()
    rec, ids = plugin.projected()
    return img, plugin.sorted_entries().copy(), rec.copy(), ids.copy()


@pytest.mark.parametrize("name", ["general", "translation"])
@pytest.mark.parametrize("mode,kw", RENDER_MODES, ids=[m for m, _ in RENDER_MODES])
@pytest.mark.parametrize("degree", TC.DEGREES)
def test_baked_cloud_renders_like_the_transformed_original(plugin, degree, mode, kw, name):
    c = TC.cloud(60_000, degree, 31 + degree, special=False)
    c.position_visibility[:, :3] *= F(0.1)
    c.position_visibility[:, 3] = 1.0
    M = B.similarity_transform((0.2, -0.1, 0.15), (0.9, 0.2, -0.3, 0.25), 1.1) if name == "general" \
        else B.similarity_transform((0.2, -0.1, 0.15))
    planes = TC.planes_of(c, "f32")
    view = B.headless_view(320, 200)
    s = B.CloudSettings(global_scale=0.25, binning_rounds=False, **kw)
    orig, baked = upload(plugin, "f32", degree, planes), upload(plugin, "f32", degree, planes)
    try:
        plugin.transform(baked, M)
        img_o, ent_o, rec_o, ids_o = _render(plugin, orig, s, view, B.CloudTransform(M))
        img_b, ent_b, rec_b, ids_b = _render(plugin, baked, s, view)
        assert len(ids_o) > 1000
        # the blend order and the record centres: bit for bit
        assert np.array_equal(ent_o, ent_b), "sorted entries"
        assert np.array_equal(ids_o, ids_b)
        assert np.array_equal(rec_o[:, :2].view(np.uint32), rec_b[:, :2].view(np.uint32)), "record centres"
        # the uv map as the quadratic form Q = U^T U of its rows (U = [[ux, uy], [vx, vy]]): a near-isotropic splat's uv
        # frame may turn freely under rounding, its form does not.  The two sides' 3D covariances differ by about 1e-6
        # relative (q_R and the products rounded apart); the projection's eigenvalues amplify that by the form's
        # condition number kappa, so each record's largest entry error is bounded by 1e-3 + 1e-5 kappa of its largest entry.
        # The OBB record's eigenvectors follow the reference's quirks (b = 0 with a != c, a NaN eigenvector), which are
        # discontinuous in the covariance: a record there may leave the bound, at most 1 in 1000 of them, and the pixels
        # below bound what it costs.
        U_o, U_b = rec_o[:, 2:6].reshape(-1, 2, 2).astype(np.float64), rec_b[:, 2:6].reshape(-1, 2, 2).astype(np.float64)
        Q_o, Q_b = U_o.transpose(0, 2, 1) @ U_o, U_b.transpose(0, 2, 1) @ U_b
        ev = np.linalg.eigvalsh(Q_o)
        kappa = ev[:, 1] / np.maximum(ev[:, 0], 1e-30)
        rel = np.abs(Q_o - Q_b).max((1, 2)) / np.maximum(np.abs(Q_o).max((1, 2)), 1e-12)
        q_out = int(np.sum(rel > 1e-3 + 1e-5 * kappa))
        col_err = np.abs(rec_o[:, 8:11] - rec_b[:, 8:11]).max()
        op_err = np.abs(rec_o[:, 11] - rec_b[:, 11]).max()
        d = np.abs(img_o - img_b)
        stats = dict(q_out=q_out, n=len(rel), col_err=col_err, op_err=op_err, px_mean=d.mean(), px_max=d.max())
        assert q_out * 1000 <= len(rel) and col_err <= 2e-4 and op_err <= 1e-6, stats
        # pixels: mean |d| <= 1e-4, each <= 2e-2 (a turned uv frame moves the corners of an OBB quad, where the weight
        # is below exp(-4.5) of the opacity)
        assert d.mean() <= 1e-4 and d.max() <= 2e-2, stats
        if mode == "3dgs_aabb":   # the conic's bbox follows the eigenvalues only: within a pixel
            bo, bb = rec_o[:, 6:8].view(np.uint32), rec_b[:, 6:8].view(np.uint32)
            for sh in (0, 16):
                e = np.abs(((bo >> sh) & 0xFFFF).astype(np.int64) - ((bb >> sh) & 0xFFFF).astype(np.int64))
                assert e.max() <= 1, "bbox"
        # the baked positions are the world positions the transformed frame computes
        p_b = plugin.positions(baked)
        assert np.array_equal(p_b[:, :3].view(np.uint32), TC.mat4_point(M, planes[0]).view(np.uint32))
    finally:
        orig.destroy(); baked.destroy()


# ---- 3. both device copies ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sel", [False, True], ids=["all", "selected"])
@pytest.mark.parametrize("layout", TC.LAYOUTS)
def test_transformed_frames_equal_fresh_upload(plugin, layout, sel):
    c = TC.cloud(30_000, 3, 41, special=False)
    c.position_visibility[:, :3] *= F(0.1)
    planes = TC.planes_of(c, layout)
    view = B.headless_view(320, 200)
    h = upload(plugin, layout, 3, planes)
    try:
        plugin.transform(h, B.similarity_transform((0.1, 0.0, -0.1), (0.8, 0.3, 0.1, -0.2), 0.9), selected=sel)
        got_planes = plugin.download_planes(h)     # (checked against the oracle above)
        fresh = upload(plugin, layout, 3, got_planes)
        fresh.aabb = h.aabb
        try:
            for mname, kw in [("3dgs", {}), ("selected", dict(draw_mode=B.DrawMode.Selected)),
                              ("depth", dict(rasterize_mode=B.RasterizeMode.Depth))]:
                s = B.CloudSettings(global_scale=0.25, binning_rounds=False, **kw)
                a, b = _render(plugin, h, s, view), _render(plugin, fresh, s, view)
                assert len(a[3]) > 100, mname
                for x, y in zip(a, b):
                    assert np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32)), mname
        finally:
            fresh.destroy()
    finally:
        h.destroy()


# ---- 4. ordering across contexts, no host synchronisation in between ---------------------------------------------
def test_queued_frames_see_exactly_the_transforms_enqueued_before_them():
    import torch

    n, w, hgt, layout = 1_000_000, 1920, 1080, "f16"
    c = B.random_gaussians_3d_seeded(n, 5)
    c.position_visibility[:, 3] = (np.random.default_rng(5).random(n) < 0.5).astype(F)
    planes = TC.planes_of(c, layout)
    s = B.CloudSettings(global_scale=0.05, binning_rounds=False)
    view = B.headless_view(w, hgt)
    M1 = B.similarity_transform((1.0, 0.5, 0.0), (0.95, 0.0, 0.3, 0.0), 1.0)
    M2 = B.similarity_transform((-2.0, 0.0, 1.0), (0.9, 0.4, 0.0, 0.1), 0.8)
    A, Bp, Cp, ref = (B.GaussianSplattingPlugin(0) for _ in range(4))
    h = upload(A, layout, 3, planes)
    try:
        # the states, as the GPU computes them, on a context of their own
        states, r = [planes], upload(ref, layout, 3, planes)
        for M, sel in ((M1, False), (M2, True)):
            ref.transform(r, M, selected=sel)
            states.append(ref.download_planes(r))
        r.destroy()
        for p in (A, Bp, Cp):
            p.render_view(h, s, view, to_host=False)
            p.render_view(h, s, view, to_host=False, asynchronous=True)
            assert p.sync()
        outs = [torch.empty((hgt, w, 4), dtype=torch.float32, device="cuda:0") for _ in range(4)]
        torch.cuda.synchronize()
        frame = lambda p, k: p.render_view_to_device(h, s, view, outs[k].data_ptr(), fmt="rgba32f", asynchronous=True)
        frame(A, 0)                          # S0
        Bp.transform(h, M1)                  # -> S1
        frame(Cp, 1)                         # S1
        Cp.transform(h, M2, selected=True)   # -> S2
        frame(A, 2)                          # S2
        frame(Bp, 3)                         # S2
        for p in (A, Bp, Cp):
            assert p.sync()
        got = [o.cpu().numpy() for o in outs]
        want = []
        for st in states:
            hr = upload(ref, layout, 3, st)
            want.append(ref.render_view(hr, s, view, fmt="rgba32f").copy())
            hr.destroy()
        for a in range(3):
            for b in range(a + 1, 3):
                assert not np.array_equal(want[a], want[b])
        for k, st in enumerate((0, 1, 2, 2)):
            assert np.array_equal(got[k].view(np.uint32), want[st].view(np.uint32)), f"frame {k} is not S{st}"
        final = A.download_planes(h)
        for g, w_ in zip(final, states[2]):
            assert np.array_equal(np.asarray(g).view(np.uint32), np.asarray(w_).view(np.uint32))
    finally:
        h.destroy()
        for p in (A, Bp, Cp, ref):
            p.destroy()


def test_transform_sees_a_particle_step_queued_on_another_context(plugin):
    other = B.GaussianSplattingPlugin(0)
    n, layout = 1_000_000, "f32"
    planes = TC.planes_of(TC.cloud(n, 3, 12, special=False), layout)
    beh = B.random_particle_behaviors(n, 12)
    h = upload(plugin, layout, 3, planes)
    parts = other.add_particles(beh)
    try:
        other.step_particles(h, parts, 0.25)
        plugin.transform(h, TC.ACCEPTED["general"])        # no sync of `other` in between
        stepped = (PO.particle_step(planes[0], beh, 0.25)[0],) + tuple(planes[1:])
        want, bound = TO.transform(layout, 3, stepped, TC.ACCEPTED["general"])
        assert_transformed(layout, 3, plugin.download_planes(h), want, bound, stepped, np.ones(n, bool), "after a step")
        assert plugin.sync() and other.sync()
    finally:
        parts.destroy(); h.destroy(); other.destroy()


# ---- 5. bounds --------------------------------------------------------------------------------------------------------
def _assert_bounds(got, want, what):
    (glo, ghi, gn), (wlo, whi, wn) = got, want
    assert gn == wn, f"{what}: count {gn} != {wn}"
    assert np.array_equal(glo, wlo) and np.array_equal(ghi, whi), f"{what}: {glo} {ghi} != {wlo} {whi}"   # (-0 == +0)


@pytest.mark.parametrize("layout", ["f32", "f16"])
def test_bounds_match_numpy(plugin, layout):
    c = TC.cloud(N, 3, 51)
    h = upload(plugin, layout, 3, TC.planes_of(c, layout))
    try:
        pos = plugin.positions(h)
        for sel in (False, True):
            _assert_bounds(plugin.bounds(h, selected=sel), TC.bounds(pos, sel), f"sel={sel}")
        plugin.set_visibility(h, np.zeros(N, F))                        # an empty selection
        lo, hi, cnt = plugin.bounds(h, selected=True)
        assert cnt == 0 and np.all(lo == np.inf) and np.all(hi == -np.inf)
        plugin.transform(h, TC.ACCEPTED["general"])                       # queued; the bounds wait for it
        _assert_bounds(plugin.bounds(h), TC.bounds(plugin.positions(h), False), "after a transform")
    finally:
        h.destroy()


def test_bounds_of_non_finite_positions_only_are_empty(plugin):
    c = TC.cloud(1000, 0, 52, special=False)
    c.position_visibility[:, 0] = np.nan
    c.position_visibility[::2, 0] = np.inf
    h = upload(plugin, "f32", 0, TC.planes_of(c, "f32"))
    try:
        lo, hi, cnt = plugin.bounds(h)
        assert cnt == 0 and np.all(lo == np.inf) and np.all(hi == -np.inf)
    finally:
        h.destroy()


def test_bounds_after_a_queued_particle_step_and_update_aabb(plugin):
    other = B.GaussianSplattingPlugin(0)
    n = 500_000
    planes = TC.planes_of(TC.cloud(n, 3, 53, special=False), "f32")
    beh = B.random_particle_behaviors(n, 53)
    h = upload(plugin, "f32", 3, planes)
    parts = other.add_particles(beh)
    try:
        other.step_particles(h, parts, 0.5)
        want_pos = PO.particle_step(planes[0], beh, 0.5)[0]
        _assert_bounds(plugin.bounds(h), TC.bounds(want_pos, False), "after a step")
        plugin.transform(h, TC.ACCEPTED["turn_z"], selected=True)
        aabb = plugin.update_aabb(h)
        want = compute_aabb(plugin.positions(h))
        for g, w in zip(aabb, want):
            assert np.array_equal(g.view(np.uint32), w.view(np.uint32))
        assert h.aabb is aabb
        assert plugin.sync() and other.sync()
    finally:
        parts.destroy(); h.destroy(); other.destroy()


def test_bounds_of_a_4d_cloud_are_its_base_positions(plugin):
    c4 = B.random_gaussians_4d_seeded(5000, 3)
    h = plugin.add_cloud(c4)
    try:
        _assert_bounds(plugin.bounds(h), TC.bounds(c4.position_visibility, False), "4D")
    finally:
        h.destroy()


# ---- 6. refusals ----------------------------------------------------------------------------------------------------
def test_refusals_change_nothing(plugin):
    lib, ctx = plugin._lib, plugin._ctx
    planes = TC.planes_of(TC.cloud(2000, 3, 61), "f16")
    h = upload(plugin, "f16", 3, planes)
    h4 = plugin.add_cloud(B.random_gaussians_4d_seeded(1000, 4))
    try:
        before, before4 = plugin.download_planes(h), plugin.download_planes(h4)
        for name, m in TC.REFUSED.items():
            for mode in (0, 1):
                cm = np.ascontiguousarray(np.asarray(m, F).T.reshape(16))
                assert lib.bgs_cloud_transform(ctx, h._h, _ptr(cm), mode) == abi.BGS_EINVAL, name
        ok = np.ascontiguousarray(TC.ACCEPTED["general"].T.reshape(16))
        assert lib.bgs_cloud_transform(ctx, h._h, _ptr(ok), 2) == abi.BGS_EINVAL
        assert lib.bgs_cloud_transform(ctx, h._h, None, 0) == abi.BGS_EINVAL
        assert lib.bgs_cloud_transform(ctx, None, _ptr(ok), 0) == abi.BGS_EINVAL
        assert lib.bgs_cloud_transform(None, h._h, _ptr(ok), 0) == abi.BGS_EINVAL
        assert lib.bgs_cloud_transform(ctx, h4._h, _ptr(ok), 0) == abi.BGS_EINVAL
        lo, hi = np.empty(3, F), np.empty(3, F)
        assert lib.bgs_cloud_bounds(ctx, h._h, 2, _ptr(lo), _ptr(hi), None) == abi.BGS_EINVAL
        assert lib.bgs_cloud_bounds(ctx, h._h, 0, None, _ptr(hi), None) == abi.BGS_EINVAL
        with pytest.raises(abi.BgsError):
            plugin.transform(h, TC.REFUSED["shear"])
        assert plugin.sync()
        for g, w in zip(plugin.download_planes(h), before):
            assert np.array_equal(np.asarray(g).view(np.uint32), np.asarray(w).view(np.uint32))
        for g, w in zip(plugin.download_planes(h4), before4):
            assert np.array_equal(np.asarray(g).view(np.uint32), np.asarray(w).view(np.uint32))
    finally:
        h4.destroy(); h.destroy()


# ---- 7. a context that never transforms keeps its launches ---------------------------------------------------------
def test_launch_counts_of_a_context_that_never_transforms(plugin):
    other = B.GaussianSplattingPlugin(0)
    c = B.random_gaussians_3d_seeded(100_000, 71)
    c.position_visibility[:, :3] *= F(0.1)
    h = plugin.add_cloud(c)
    s = B.CloudSettings(global_scale=0.25, binning_rounds=False)
    view = B.headless_view(320, 200)
    try:
        plugin.render_view(h, s, view)
        before = plugin.last_launch_count
        other.transform(h, B.similarity_transform((0.01, 0.0, 0.0)))
        plugin.render_view(h, s, view)
        assert plugin.last_launch_count == before
        other.bounds(h)
        plugin.render_view(h, s, view)
        assert plugin.last_launch_count == before
        assert other.sync()
    finally:
        h.destroy(); other.destroy()
