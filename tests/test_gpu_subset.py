"""bgs_cloud_subset and bgs_cloud_download_* on the GPU, for the f32, f16 and precomputed-covariance layouts: downloads of
fresh uploads equal the upload arrays bit for bit; selection-mode subsets of every tests/subset_cases.py lane (set by
set_visibility, select_sparse and select_in_mesh) and index-mode subsets equal the host subset bit for bit; frames of
a subset equal frames of a fresh upload of the host subset; the ordering against queued particle steps, the debug
hooks and destroyed sources; 6 M gaussians; and the C++ host's save_selection against Python's."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import subset_cases as S
from bevy_gaussian_splatting_b200 import abi

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAYOUTS = ["f32", "f16", "cov"]


@pytest.fixture(scope="module")
def plugin():
    p = B.GaussianSplattingPlugin(0)
    yield p
    p.destroy()


def add(plugin, cloud, layout):
    return plugin.add_cloud(cloud, f16=layout == "f16", precompute_covariance=layout == "cov")


def upload_planes(cloud, layout):
    """The arrays the layout's upload call takes."""
    if layout == "f32":
        return cloud.position_visibility, cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity
    src = cloud.precomputed_covariance() if layout == "cov" else cloud
    return (cloud.position_visibility, *src.pack_f16())


def assert_planes(got, want, what=""):
    assert len(got) == len(want), what
    for k, (g, w) in enumerate(zip(got, want)):
        g, w = np.ascontiguousarray(g), np.ascontiguousarray(w)
        assert g.shape == w.shape, (what, k, g.shape, w.shape)
        if not np.array_equal(g.view(np.uint32), w.view(np.uint32)):
            bad = np.flatnonzero((g.view(np.uint32) != w.view(np.uint32)).any(axis=1))
            raise AssertionError(f"{what}: plane {k} differs at {len(bad)} gaussians, first {bad[:8]}")


def cloud_with_vis(vis, seed=0):
    c = B.random_gaussians_3d_seeded(len(vis), seed)
    c.position_visibility[:, 3] = vis
    return c


# ---- 1. round trip ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("n", [1, 31, 32, 33, 1000, 200_000])
def test_download_of_fresh_upload_is_the_upload(plugin, layout, n):
    cloud = B.random_gaussians_3d_seeded(n, n % 5)
    h = add(plugin, cloud, layout)
    try:
        assert_planes(plugin.download_planes(h), upload_planes(cloud, layout), f"{layout} n={n}")
        d = plugin.download(h)
        want = cloud if layout == "f32" else B.PlanarGaussian3d.from_f16(*upload_planes(cloud, layout))
        assert_planes([d.position_visibility, d.spherical_harmonic, d.rotation, d.scale_opacity],
                      [want.position_visibility, want.spherical_harmonic, want.rotation, want.scale_opacity], "download()")
    finally:
        h.destroy()


# ---- 2. selection mode --------------------------------------------------------------------------------------------
def selection_subset(plugin, h, cloud, layout, vis, what):
    idx = np.flatnonzero(S.kept(vis))
    out, n = C.c_void_p(), C.c_uint32(12345)
    plugin._check(plugin._lib.bgs_cloud_subset(plugin._ctx, h._h, None, 0, C.byref(out), C.byref(n)))
    if len(idx) == 0:
        assert not out and n.value == 0, what
        assert plugin.subset(h) is None
        return
    assert out and n.value == len(idx), what
    plugin._lib.bgs_cloud_destroy(out)
    sub = plugin.subset(h)
    try:
        planes = [p.copy() for p in upload_planes(cloud, layout)]
        planes[0][:, 3] = vis
        assert sub.n == len(idx) and sub.f16 == h.f16 and sub.precompute_covariance == h.precompute_covariance
        assert_planes(plugin.download_planes(sub), [p[idx] for p in planes], what)
        lo, hi = B.gaussian.compute_aabb(planes[0][idx])
        assert np.array_equal(sub.aabb[0], lo) and np.array_equal(sub.aabb[1], hi)
    finally:
        sub.destroy()


CASES = S.cases()


@pytest.mark.parametrize("layout", LAYOUTS)
def test_selection_mode_set_visibility(plugin, layout):
    for case in CASES:
        vis = case["vis"]
        cloud = cloud_with_vis(np.ones(len(vis), np.float32), len(vis) % 3)
        h = add(plugin, cloud, layout)
        try:
            plugin.set_visibility(h, vis)
            assert np.array_equal(plugin.visibility(h).view(np.uint32), vis.view(np.uint32))
            selection_subset(plugin, h, cloud, layout, vis, f"{layout} {case['name']}")
        finally:
            h.destroy()


def cube(lo, hi):
    v = np.array([[x, y, z] for x in (lo, hi) for y in (lo, hi) for z in (lo, hi)], np.float32)
    f = [(0, 1, 3), (0, 3, 2), (4, 6, 7), (4, 7, 5), (0, 4, 5), (0, 5, 1), (2, 3, 7), (2, 7, 6), (0, 2, 6), (0, 6, 4),
         (1, 5, 7), (1, 7, 3)]
    return v, np.array(f, np.uint32)


@pytest.mark.parametrize("layout", LAYOUTS)
def test_selection_mode_select_sparse_and_in_mesh(plugin, layout):
    cloud = B.random_gaussians_3d_seeded(100_003, 9)
    cloud.position_visibility[:, :3] *= np.float32(0.05)
    h = add(plugin, cloud, layout)
    try:
        for what, select in (("sparse", lambda: plugin.select_sparse(h, B.SparseSelect(0.02, 3))),
                             ("sparse_none", lambda: plugin.select_sparse(h, B.SparseSelect(0.02, 0))),
                             ("sparse_all", lambda: plugin.select_sparse(h, B.SparseSelect(0.0, 1))),
                             ("mesh", lambda: plugin.select_in_mesh(h, *cube(-0.4, 0.4))),
                             ("mesh_none", lambda: plugin.select_in_mesh(h, *cube(5.0, 6.0)))):
            count = select()
            vis = plugin.visibility(h)
            assert S.kept(vis).sum() == count, what
            selection_subset(plugin, h, cloud, layout, vis, f"{layout} {what}")
    finally:
        h.destroy()


# ---- 3. index mode ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", LAYOUTS)
def test_index_mode(plugin, layout):
    n = 5000
    cloud = B.random_gaussians_3d_seeded(n, 13)
    cloud.position_visibility[:, 3] = np.resize(S.cases()[0]["vis"], n)
    h = add(plugin, cloud, layout)
    rng = np.random.default_rng(3)
    try:
        for what, idx in (("random_repeats", rng.integers(0, n, 3000)), ("k1", np.array([n - 1])), ("k1_first", np.array([0])),
                          ("k_gt_n", rng.integers(0, n, 3 * n + 7)), ("reversed", np.arange(n)[::-1]),
                          ("all_same", np.full(777, 42))):
            sub = plugin.subset(h, idx)
            try:
                assert sub.n == len(idx)
                assert_planes(plugin.download_planes(sub), [p[idx] for p in upload_planes(cloud, layout)], f"{layout} {what}")
            finally:
                sub.destroy()
    finally:
        h.destroy()


def test_refusals_create_nothing(plugin):
    lib, ctx = plugin._lib, plugin._ctx
    cloud = B.random_gaussians_3d_seeded(1000, 2)
    h = plugin.add_cloud(cloud)
    hf = plugin.add_cloud(cloud, f16=True)
    try:
        before = len(plugin.download_planes(h)[0])
        idx = np.arange(1000, dtype=np.uint32)
        bad = idx.copy(); bad[500] = 1000
        ip = idx.ctypes.data_as(C.c_void_p)
        bp = bad.ctypes.data_as(C.c_void_p)
        buf = [np.empty((1000, w), np.float32) for w in (4, 48, 4, 4)]
        bptr = [b.ctypes.data_as(C.c_void_p) for b in buf]

        def refused(call, status=abi.BGS_EINVAL):
            out, n = C.c_void_p(1), C.c_uint32(77)
            assert call(C.byref(out), C.byref(n)) == status
            assert not out.value and n.value == 77

        refused(lambda o, n: lib.bgs_cloud_subset(ctx, h._h, bp, 1000, o, n))               # an index >= n
        refused(lambda o, n: lib.bgs_cloud_subset(ctx, h._h, ip, 0, o, n))                  # k == 0
        refused(lambda o, n: lib.bgs_cloud_subset(ctx, h._h, ip, 1 << 30, o, n))            # k >= 2^30
        refused(lambda o, n: lib.bgs_cloud_subset(ctx, h._h, None, 5, o, n))                # selection mode with k != 0
        refused(lambda o, n: lib.bgs_cloud_subset(ctx, None, ip, 10, o, n))
        assert lib.bgs_cloud_subset(None, h._h, ip, 10, None, None) == abi.BGS_EINVAL
        assert lib.bgs_cloud_subset(ctx, h._h, ip, 10, None, None) == abi.BGS_EINVAL
        with pytest.raises(abi.BgsError):
            plugin.subset(h, bad)
        with pytest.raises(abi.BgsError):
            plugin.subset(h, np.array([], np.uint32))
        # downloads: nulls and the wrong layout
        assert lib.bgs_cloud_download_f32(None, h._h, *bptr) == abi.BGS_EINVAL
        assert lib.bgs_cloud_download_f32(ctx, None, *bptr) == abi.BGS_EINVAL
        for k in range(4):
            args = list(bptr); args[k] = None
            assert lib.bgs_cloud_download_f32(ctx, h._h, *args) == abi.BGS_EINVAL
        assert lib.bgs_cloud_download_f32(ctx, hf._h, *bptr) == abi.BGS_EINVAL
        assert lib.bgs_cloud_download_f16(ctx, h._h, *bptr[:3]) == abi.BGS_EINVAL
        for k in range(3):
            args = list(bptr[:3]); args[k] = None
            assert lib.bgs_cloud_download_f16(ctx, hf._h, *args) == abi.BGS_EINVAL
        assert before == 1000
        assert_planes(plugin.download_planes(h), upload_planes(cloud, "f32"), "after refusals")
    finally:
        h.destroy(); hf.destroy()


# ---- 4. frames of a subset ----------------------------------------------------------------------------------------
SETTINGS_2 = [("3dgs_obb", {}), ("3dgs_aabb", dict(aabb=True)), ("2dgs", dict(gaussian_mode=B.GaussianMode.Gaussian2d)),
              ("selected", dict(draw_mode=B.DrawMode.Selected)),
              ("highlight_selected", dict(draw_mode=B.DrawMode.HighlightSelected)),
              ("depth", dict(rasterize_mode=B.RasterizeMode.Depth)), ("position", dict(rasterize_mode=B.RasterizeMode.Position))]


def frame_and_records(plugin, h, settings, view):
    img = plugin.render_view(h, settings, view, fmt="rgba32f")
    rec, ids = plugin.projected()
    return img.copy(), rec.copy(), ids.copy()


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("mode", ["selection", "index"])
def test_subset_frames_equal_fresh_upload(plugin, layout, mode):
    n = 40_000
    cloud = B.random_gaussians_3d_seeded(n, 21)
    cloud.position_visibility[:, :3] *= np.float32(0.1)
    rng = np.random.default_rng(21)
    # kept ones carry visibilities on both sides of 0.5 afterwards only in index mode; selection mode keeps w >= 0.5
    cloud.position_visibility[:, 3] = rng.choice(np.array([0.0, 0.25, 0.5, 0.75, 1.0], np.float32), n)
    view = B.headless_view(320, 200)
    h = add(plugin, cloud, layout)
    idx = np.flatnonzero(S.kept(cloud.position_visibility[:, 3])) if mode == "selection" else rng.integers(0, n, n // 2)
    sub = plugin.subset(h) if mode == "selection" else plugin.subset(h, idx)
    host = cloud.subset(idx)
    fresh = add(plugin, host, layout)
    fresh.aabb = sub.aabb
    try:
        assert np.array_equal(sub.aabb[0], host.compute_aabb()[0]) and np.array_equal(sub.aabb[1], host.compute_aabb()[1])
        for name, kw in SETTINGS_2:
            if layout == "cov" and name == "2dgs":
                continue
            s = B.CloudSettings(global_scale=0.25, binning_rounds=False, **kw)
            got = frame_and_records(plugin, sub, s, view)
            want = frame_and_records(plugin, fresh, s, view)
            assert len(got[2]) > 100, name
            assert np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32)), f"{name} frame"
            assert np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32)), f"{name} records"
            assert np.array_equal(got[2], want[2]), name
    finally:
        fresh.destroy(); sub.destroy(); h.destroy()


# ---- 5. ordering --------------------------------------------------------------------------------------------------
def test_subset_sees_steps_queued_on_another_context(plugin):
    from particle_oracle import particle_oracle as PO

    other = B.GaussianSplattingPlugin(0)
    n = 300_000
    cloud = B.random_gaussians_3d_seeded(n, 7)
    cloud.position_visibility[:, 3] = np.random.default_rng(7).uniform(0, 1, n).astype(np.float32)
    beh = B.random_particle_behaviors(n, 7)
    beh["velocity"][:, 3] *= np.float32(8)            # the visibility lane moves across 0.5 too
    h = plugin.add_cloud(cloud, f16=True)
    parts = other.add_particles(beh)
    try:
        for _ in range(3):
            other.step_particles(h, parts, 1 / 30)
        sub = plugin.subset(h)                       # no sync in between
        sub_i = plugin.subset(h, np.arange(n)[::-1])
        pos = cloud.position_visibility
        for _ in range(3):
            pos, beh = PO.particle_step(pos, beh, 1 / 30)
        idx = np.flatnonzero(S.kept(pos[:, 3]))
        assert 0 < len(idx) < n and not np.array_equal(S.kept(pos[:, 3]), S.kept(cloud.position_visibility[:, 3]))
        try:
            sh, rso = cloud.pack_f16()
            assert_planes(plugin.download_planes(sub), [pos[idx], sh[idx], rso[idx]], "selection after steps")
            r = np.arange(n)[::-1]
            assert_planes(plugin.download_planes(sub_i), [pos[r], sh[r], rso[r]], "index after steps")
        finally:
            sub.destroy(); sub_i.destroy()
        other.step_particles(h, parts, 1 / 30)
        pos, beh = PO.particle_step(pos, beh, 1 / 30)
        assert np.array_equal(plugin.download_planes(h)[0].view(np.uint32), pos.view(np.uint32))
        assert other.sync()
    finally:
        parts.destroy(); h.destroy(); other.destroy()


def test_debug_hooks_keep_the_last_frame(plugin):
    cloud = B.random_gaussians_3d_seeded(30_000, 4)
    cloud.position_visibility[::3, 3] = 0
    view = B.headless_view(320, 200)
    s = B.CloudSettings(global_scale=0.25, binning_rounds=False)
    h = plugin.add_cloud(cloud)
    try:
        plugin.render_view(h, s, view)
        fs0 = bytes(plugin.frame_stats())
        rec0, ids0 = plugin.projected()
        st0 = plugin.sorted_entries().copy()
        sub = plugin.subset(h)
        sub2 = plugin.subset(h, np.arange(100))
        plugin.download(h); plugin.download(sub)
        assert bytes(plugin.frame_stats()) == fs0
        rec1, ids1 = plugin.projected()
        assert np.array_equal(rec0.view(np.uint32), rec1.view(np.uint32)) and np.array_equal(ids0, ids1)
        assert np.array_equal(st0, plugin.sorted_entries())
        plugin.stage_times_us()
        sub.destroy(); sub2.destroy()
        plugin.render_view(h, s, view)
        assert plugin.last_launch_count == 6
    finally:
        h.destroy()


def test_subset_outlives_its_source_and_its_context():
    cloud = B.random_gaussians_3d_seeded(10_000, 8)
    cloud.position_visibility[1::2, 3] = 0
    idx = np.flatnonzero(S.kept(cloud.position_visibility[:, 3]))
    a, b = B.GaussianSplattingPlugin(0), B.GaussianSplattingPlugin(0)
    try:
        h = a.add_cloud(cloud, f16=True)
        sub = a.subset(h)
        h.destroy()
        a.destroy()                                   # the context that made it
        want = [p[idx] for p in upload_planes(cloud, "f16")]
        assert_planes(b.download_planes(sub), want, "after source and context destroyed")
        sub2 = b.subset(sub, np.arange(sub.n)[::-1])
        img = b.render_view(sub, B.CloudSettings(global_scale=0.25), B.headless_view(160, 100))
        assert np.isfinite(img).all()
        assert_planes(b.download_planes(sub2), [p[::-1] for p in want], "subset of a subset")
        sub2.destroy()
        sub.destroy()
    finally:
        a.destroy(); b.destroy()


def test_launch_counts_unchanged(plugin):
    view = B.headless_view(320, 200)
    s = B.CloudSettings(global_scale=0.25, binning_rounds=False)
    sd = B.CloudSettings(global_scale=0.25, binning_rounds=False, rasterize_mode=B.RasterizeMode.Depth)
    h = plugin.add_cloud(B.random_gaussians_3d_seeded(20000, 4))
    sub = plugin.subset(h)
    try:
        for c in (h, sub):
            plugin.render_view(c, s, view)
            assert plugin.last_launch_count == 6
            plugin.render_view(c, sd, view)
            assert plugin.last_launch_count == 7
    finally:
        sub.destroy(); h.destroy()


# ---- 6. scale -----------------------------------------------------------------------------------------------------
def test_six_million(plugin):
    n = 6_000_000
    cloud = B.random_gaussians_3d_seeded(n, 0)
    vis = (np.random.default_rng(0).random(n) < 0.5).astype(np.float32)
    h = plugin.add_cloud(cloud, f16=True)
    try:
        plugin.set_visibility(h, vis)
        idx = np.flatnonzero(vis)
        sub = plugin.subset(h)
        try:
            planes = [p.copy() for p in upload_planes(cloud, "f16")]
            planes[0][:, 3] = vis
            assert_planes(plugin.download_planes(sub), [p[idx] for p in planes], "C3 f16 50 %")
        finally:
            sub.destroy()
    finally:
        h.destroy()
    h = plugin.add_cloud(cloud)
    try:
        r = np.arange(n)[::-1]
        sub = plugin.subset(h, r)
        try:
            assert_planes(plugin.download_planes(sub), [p[r] for p in upload_planes(cloud, "f32")], "C3 f32 reversed")
        finally:
            sub.destroy()
    finally:
        h.destroy()


# ---- 7. the C++ host ----------------------------------------------------------------------------------------------
CPP = r"""
#include <cstdio>
#include <fstream>
#include "bgs.hpp"
// argv: cloud.bin (u64 n, then the four f32 planes), selection.bin (u64 k, then k u32 indices), out.gcloud
int main(int argc, char** argv) {
    if (argc != 4) return 2;
    std::ifstream in(argv[1], std::ios::binary);
    uint64_t n = 0;
    in.read((char*)&n, 8);
    bgs::PlanarGaussian3d c;
    c.position_visibility.resize(n * 4); c.spherical_harmonic.resize(n * 48); c.rotation.resize(n * 4); c.scale_opacity.resize(n * 4);
    for (std::vector<float>* p : {&c.position_visibility, &c.spherical_harmonic, &c.rotation, &c.scale_opacity})
        in.read((char*)p->data(), p->size() * 4);
    std::ifstream si(argv[2], std::ios::binary);
    uint64_t k = 0;
    si.read((char*)&k, 8);
    std::vector<uint32_t> sel(k);
    si.read((char*)sel.data(), k * 4);
    bgs::GaussianSplattingPlugin plugin(0);
    bgs::PlanarGaussian3dHandle h = plugin.add_cloud(c);
    plugin.apply_selection(h, sel);
    const uint32_t saved = plugin.save_selection(h, argv[3]);
    std::printf("saved=%u\n", saved);
    return 0;
}
"""


def test_cpp_host_save_selection_matches_python(plugin, tmp_path):
    n = 20_000
    cloud = B.random_gaussians_3d_seeded(n, 17)
    sel = np.sort(np.random.default_rng(17).choice(n, 6000, replace=False)).astype(np.uint32)
    with open(tmp_path / "cloud.bin", "wb") as f:
        f.write(np.uint64(n).tobytes())
        for p in (cloud.position_visibility, cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity):
            f.write(p.tobytes())
    with open(tmp_path / "sel.bin", "wb") as f:
        f.write(np.uint64(len(sel)).tobytes() + sel.tobytes())
    src = tmp_path / "save_selection.cpp"
    src.write_text(CPP)
    exe = tmp_path / "save_selection"
    libdir = os.path.join(ROOT, "bevy_gaussian_splatting_b200")
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe),
                    "-L", libdir, "-lbgs", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True, text=True)
    out = subprocess.run([str(exe), str(tmp_path / "cloud.bin"), str(tmp_path / "sel.bin"), str(tmp_path / "cpp.gcloud")],
                         check=True, capture_output=True, text=True).stdout
    assert f"saved={len(sel)}" in out
    h = plugin.add_cloud(cloud)
    try:
        plugin.apply_selection(h, sel)
        assert plugin.save_selection(h, tmp_path / "py.gcloud") == len(sel)
    finally:
        h.destroy()
    a, b = B.read_gcloud(tmp_path / "cpp.gcloud"), B.read_gcloud(tmp_path / "py.gcloud")
    want = cloud.subset(sel)
    want.position_visibility[:, 3] = 1.0
    for x, y, z in ((a.position_visibility, b.position_visibility, want.position_visibility),
                    (a.spherical_harmonic, b.spherical_harmonic, want.spherical_harmonic),
                    (a.rotation, b.rotation, want.rotation), (a.scale_opacity, b.scale_opacity, want.scale_opacity)):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
        assert np.array_equal(x.view(np.uint32), z.view(np.uint32))


# ---- save_selection (Python host) -----------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", LAYOUTS)
def test_save_selection(plugin, tmp_path, layout):
    cloud = B.random_gaussians_3d_seeded(3000, 6)
    vis = np.resize(S.cases()[0]["vis"], 3000)
    h = add(plugin, cloud, layout)
    try:
        plugin.set_visibility(h, vis)
        if layout == "cov":
            with pytest.raises(ValueError):
                plugin.save_selection(h, tmp_path / "x.gcloud")
            assert not os.path.exists(tmp_path / "x.gcloud")
            return
        k = plugin.save_selection(h, tmp_path / "sel.gcloud")
        idx = np.flatnonzero(S.kept(vis))
        assert k == len(idx)
        back = B.read_gcloud(tmp_path / "sel.gcloud")
        host = cloud if layout == "f32" else cloud.rounded_to_f16()
        want = host.subset(idx)
        want.position_visibility[:, 3] = vis[idx]
        for x, y in ((back.position_visibility, want.position_visibility), (back.spherical_harmonic, want.spherical_harmonic),
                     (back.rotation, want.rotation), (back.scale_opacity, want.scale_opacity)):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
        assert plugin.save_selection(h, tmp_path / "sel.ply") == k
        assert len(B.load_cloud(tmp_path / "sel.ply")) == k + 32 - k % 32
        plugin.set_visibility(h, np.zeros(3000, np.float32))
        with pytest.raises(ValueError):
            plugin.save_selection(h, tmp_path / "none.gcloud")
        assert not os.path.exists(tmp_path / "none.gcloud")
    finally:
        h.destroy()
