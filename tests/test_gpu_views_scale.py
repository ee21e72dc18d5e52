"""bgs_render_views and bgs_render_views_aux at the sizes where binning, the tile-id sort, key-gen and the per-view Depth
range leave their small-frame paths (inputs: views_scale_cases.py).  Every views frame is held to three references:
* per-view bytes: view i's frame is bgs_render_entities_ex's (bgs_render_entities_aux's) frame of view i on the same
  context, byte for byte, in RGBA32F and RGBA8-sRGB, into host and device targets, some cases with per-view depth
  buffers; quad-uv lists also against the single-view frame's raster2_kernel and binning-round paths;
* restricted hooks: the joint frame's sorted entries, records, ids, splat depths and tile lists restricted to view i are
  view i's single-view hooks (views_scale_cases.check_restricted);
* the entity oracle: some views of every case, sorted entries, n_vis, n_pairs, tile ranges and entries bit for bit,
  pixels within 1e-3.
Each case asserts through kernel_paths that it reached the path it exists for.  The tests without the gpu mark pin the
new rules and check that each construction has the shape it is built for.
Runtime on an H100 80GB HBM3 (700 W): about 45 s for the file."""
import dataclasses
import os
import re
import subprocess

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import kernel_paths as KP
import views_cases as V
import views_scale_cases as VS
from bevy_gaussian_splatting_b200 import abi

gpu = pytest.mark.gpu
M = B.RasterizeMode
NO_CHUNKS, CHUNKS, ASYNC = abi.BGS_FLAG_NO_CHUNKS, abi.BGS_FLAG_CHUNKS, abi.BGS_FLAG_ASYNC


def _h100():
    sm = KP.device_sm_count()
    if sm != KP.H100_SMS:
        pytest.skip(f"the paths are planned for {KP.H100_SMS} SMs, this device has {sm}")
    return sm


def _per_view(p, sc, vs, got_outs, fmt, device, flags=0, depths=None, aux=False):
    """Each view's single-view frame (with `flags`) against the views frame's outputs; -> each view's hooks."""
    wants = []
    for i, v in enumerate(vs):
        z = None if depths is None else depths[i]
        if aux:
            want = [VS.target(v, fmt, device) for _ in range(3)]
            VS.ok(p, sc.aux(v, want, fmt, flags, z, device))
            for f in range(3):
                assert VS.as_bytes(got_outs[i][f]) == VS.as_bytes(want[f]), (fmt, device, i, f)
        else:
            want = VS.target(v, fmt, device)
            VS.ok(p, sc.ex(v, want, fmt, flags, z, device))
            assert VS.as_bytes(got_outs[i]) == VS.as_bytes(want), (fmt, device, i)
        wants.append(VS.hooks(p, z is not None))
    return wants


def _views(p, sc, vs, fmt, device, flags=0, depths=None, aux=False):
    if aux:
        outs = [[VS.target(v, fmt, device) for _ in range(3)] for v in vs]
        VS.ok(p, sc.views_aux(vs, outs, fmt, flags, depths, device))
    else:
        outs = [VS.target(v, fmt, device) for v in vs]
        VS.ok(p, sc.views(vs, outs, fmt, flags, depths, device))
    if flags & ASYNC:
        assert p.sync()
    return outs


def _full_check(p, sc, vs, runs, depths=None, oracle_views=(), aux=False):
    """runs: [(fmt, device, flags)].  Each run's views frame against the per-view frames; the first run's joint hooks
    restricted to each view against that view's hooks; the oracle on `oracle_views` (the first f32 host run).  -> the first
    run's joint hooks and outputs."""
    first, oracle_done = None, False
    for fmt, device, flags in runs:
        outs = _views(p, sc, vs, fmt, device, flags, depths, aux)
        got = VS.hooks(p, depths is not None)
        wants = _per_view(p, sc, vs, outs, fmt, device, NO_CHUNKS, depths, aux)
        if first is None:
            VS.check_restricted(got, wants, vs)
            first = (got, outs)
        if fmt == "f32" and not device and not oracle_done:
            oracle_done = True
            for i in oracle_views:
                orc = sc.oracle_frame(vs[i], None if depths is None else depths[i])
                VS.check_oracle(wants[i], outs[i][0] if aux else outs[i], orc)
    return first


# ---------------------------------------------------------------------------------------------------------------------
# tests without a GPU: the rules and the constructions

def test_new_rules_table():
    assert KP.views_tiles([(16, 16), (17, 17), (1, 1)]) == [0, 1, 5, 6]
    assert KP.views_bin_grid(132, False) == 396 and KP.views_bin_grid(132, True) == 132
    assert KP.views_bin_grid(132, False, views_per_sm=2) == 264
    assert [KP.depth_range_views_grid(h) for h in (0, 1, 256, 257, 1025, 135_168, 10**7)] == [1, 1, 1, 2, 5, 528, 528]
    assert KP.depth_range_views_passes(1, 1) == 1 and KP.depth_range_views_passes(257, 1) == 2
    assert KP.depth_range_views_passes(48_000, 5) == 38
    assert KP.depth_range_views_cta(255, 5) == 0 and KP.depth_range_views_cta(256, 5) == 1 and KP.depth_range_views_cta(1280, 5) == 0
    # warp_first_miss: one round when the answer is 0 or the run has at most 32 entries, more past that
    assert KP.warp_first_miss_rounds(0, 0) == 0 and KP.warp_first_miss_rounds(32, 7) == 1 and KP.warp_first_miss_rounds(5000, 0) == 1
    assert KP.warp_first_miss_rounds(64, 64) == 2 and KP.warp_first_miss_rounds(6000, 2500) >= 3
    for length in (1, 31, 33, 1000, 1025, 6000):
        for first in sorted({0, 1, length // 2, length - 1, length}):
            KP.warp_first_miss_rounds(length, first)   # (asserts it ends at `first`)


def test_tile_sets_have_their_totals_and_passes():
    for name, sizes in VS.TILE_SETS.items():
        total = KP.views_tiles(sizes)[-1]
        assert total == VS.TILE_TOTALS[name] and KP.pair_passes(total) == VS.TILE_PASSES[name], name
        assert len(VS.tile_set(name)) == len(sizes)
    t0 = KP.views_tiles(VS.TILE_SETS["t65536"])
    assert -(-VS.WIDE[0] // 16) == 4096 and t0[1] == 8160 and t0[2] - t0[1] == 8192   # the wide view between 1080p views
    assert KP.views_tiles(VS.TILE_SETS["t9x1080"])[8] < 65536   # view 8 holds the tile ids from 2^16 on


def test_footprint_views_and_cloud():
    vs = VS.footprint_views()
    assert [-(-v.width // 16) for v in vs] == [1, 31, 32, 33, 120]
    assert KP.large_split_parts(5 * 4, KP.views_bin_grid(132, False)) == 16
    assert KP.large_split_parts(5 * 4 - 2, KP.views_bin_grid(132, True)) == 16
    assert KP.large_split_parts(40, KP.views_bin_grid(132, True)) == 8
    assert KP.large_split_parts(4 * 200 + 90, KP.views_bin_grid(132, False)) == 1
    c = VS.footprint_cloud(4)
    assert len(c.position_visibility) == VS.B_N + 4


def test_footprint_classes_against_the_oracle(oracle):
    """Every view of B has tiny, medium and large footprints (from the entity oracle's bboxes)."""
    from entity_oracle import entity_oracle as EO
    import entity_cases as E

    for n_large, large_per_view in ((4, (1, 4)), (200, (60, 200))):
        c = VS.footprint_cloud(n_large)
        st = B.CloudSettings()
        u = B.GaussianSplattingPlugin.cloud_uniform(st, None, c.compute_aabb())
        total = 0
        for v in VS.footprint_views():
            o = EO.frame([E.oracle_entry(c, "f32", u, st)], v.to_abi(), [st.to_abi()], [1], want_image=False)
            fc = VS.footprint_counts(o["records"], o["rank_to_id"], 1 << 30, 1)[0]
            assert fc["tiny"] > 0 and fc["medium"] > 0 and large_per_view[0] <= fc["large"] <= large_per_view[1], (n_large, fc)
            total += fc["large"]
        parts = KP.large_split_parts(total, KP.views_bin_grid(132, False))
        assert parts == (16 if n_large == 4 else 1), (total, parts)


def test_many_view_and_keygen_sizes():
    vs = VS.many_views(64)
    assert {(v.width, v.height) for v in vs} >= {(1, 1), (16, 16), (17, 17)}
    grid = KP.scene_keygen_grid(queued=True)
    assert KP.keygen_multi_chunk(64 * VS.D_N, grid) and KP.keygen_multi_chunk(8 * 8 * VS.D_N8, grid)
    assert not KP.keygen_multi_chunk(VS.D_N, grid)
    # C: 8 views of C_N could exceed the synchronous views binning grid's single sub-tile; the GPU test checks n_visible
    assert len(VS.C_SIZES) * VS.C_N > KP.views_bin_grid(132, False) * KP.BIN_SUBTILE_MAX


def test_depth_range_cloud_runs():
    """G's near views: visible runs of thousands whose first departures lie deep inside, forwards and backwards, so each
    warp_first_miss search loops more than once."""
    n = VS.G_NEAR
    run = np.array([g for g in range(n) if g not in VS.MARKERS or g == VS.G_FAR_MISS])
    lo, hi = VS.first_misses(run, n)
    assert (lo, hi) == (VS.G_FIRST_MISS, n - 1 - VS.G_LAST_MISS)
    assert len(run) > 32 * 32 and KP.warp_first_miss_rounds(len(run), lo) > 1 and KP.warp_first_miss_rounds(len(run), hi) > 1


def _cuobjdump():
    import shutil

    return shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")


def test_bin_views_kernel_occupancy_matches_the_pinned_fit():
    """KP.BIN_VIEWS_CTAS_PER_SM_FIT against the built bin_emit_views_kernel (sm_90's allocation rules, as
    test_gpu_binning's test of bin_emit_coop_kernel)."""
    lib = abi.LIB_PATH
    if not os.path.exists(lib):
        pytest.skip("libbgs.so is not built")
    out = subprocess.run([_cuobjdump(), "--dump-resource-usage", lib], check=True, capture_output=True, text=True).stdout
    m = re.search(r"Function \S*bin_emit_views_kernel\S*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", out)
    assert m, "bin_emit_views_kernel not found in libbgs.so"
    regs, stack, shared, local = map(int, m.groups())
    warp_regs = -(-regs * 32 // 256) * 256
    fit = min((65536 // warp_regs) // (256 // 32), (228 * 1024) // (shared + 1024), 2048 // 256, 32)
    assert fit == KP.BIN_VIEWS_CTAS_PER_SM_FIT, (regs, shared, fit)
    assert stack == 0 and local == 0


# ---------------------------------------------------------------------------------------------------------------------
# A: tile-id sort passes and tile-id width

A_RUNS = {"t256": [("f32", False, 0), ("u8", True, 0)], "t257": [("f32", False, 0), ("u8", False, 0)],
          "t65536": [("f32", False, 0), ("u8", True, 0)], "t65537": [("f32", False, 0), ("u8", True, 0)],
          "t9x1080": [("f32", False, 0), ("u8", True, 0)]}
A_ORACLE = {"t256": (0, 1, 2), "t257": (1, 2, 3), "t65536": (1,), "t65537": (1, 8), "t9x1080": (8,)}


@gpu
@pytest.mark.parametrize("name", list(VS.TILE_SETS))
def test_a_tile_sort_passes(name):
    _h100()
    vs = VS.tile_set(name)
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = VS.Scene(p, VS.quad_entities(VS.room_cloud(20_000, 11)))
        depths = [VS.depth_buffer(v, 40 + i) for i, v in enumerate(vs)] if name in ("t257", "t65537") else None
        got, _ = _full_check(p, sc, vs, A_RUNS[name], depths, A_ORACLE[name])
        total = got["stats"].tiles_x
        assert total == VS.TILE_TOTALS[name] and KP.pair_passes(total) == VS.TILE_PASSES[name]
        ranges = got["ranges"].astype(np.int64)
        for i, (a, b) in enumerate(zip(KP.views_tiles([(v.width, v.height) for v in vs])[:-1],
                                       KP.views_tiles([(v.width, v.height) for v in vs])[1:])):
            assert (ranges[a:b, 1] > ranges[a:b, 0]).any(), ("a view with no pairs", i)
        if total > 65536:
            assert (ranges[65536:, 1] > ranges[65536:, 0]).any(), "tile ids >= 2^16 must hold pairs"
    finally:
        p.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# B: footprint classes under VIEWS

@gpu
@pytest.mark.parametrize("n_large", [4, 200])
def test_b_footprint_classes(n_large):
    _h100()
    vs = VS.footprint_views()
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = VS.Scene(p, [(VS.footprint_cloud(n_large), "f32", None, B.CloudSettings())])
        depths = [VS.depth_buffer(v, 60 + i) for i, v in enumerate(vs)] if n_large == 4 else None
        for queued in (False, True):
            flags = ASYNC if queued else 0
            runs = [("f32", False, flags), ("u8", True, flags)]
            got, outs = _full_check(p, sc, vs, runs, depths, (1, 2, 3) if not queued else ())
            counts = VS.footprint_counts(got["records"], got["ids"], sc.n_view, len(vs))
            for i, fc in enumerate(counts):
                assert fc["tiny"] > 0 and fc["medium"] > 0 and fc["large"] > 0, (i, fc)
            n_big = sum(fc["large"] for fc in counts)
            parts = KP.large_split_parts(n_big, KP.views_bin_grid(KP.H100_SMS, queued))
            assert parts == {(4, False): 16, (4, True): 16, (200, False): 1, (200, True): 1}[(n_large, queued)], (n_big, parts)
            if queued:
                continue
            # the single-view frames on their own quad-uv paths: raster2_kernel<false, Z> after a frame of large
            # footprints, and binning rounds (raster2_kernel<true, Z>): the same bytes as the views frame's view
            host = [VS.as_host(o) for o in outs]
            for i, v in enumerate(vs):
                # (the hints come from the previous frame: the 1080p view's, with many pairs per visible splat)
                VS.ok(p, sc.ex(vs[4], VS.target(vs[4], "f32", False), "f32", NO_CHUNKS, None if depths is None else depths[4]))
                fs = p.frame_stats()
                assert KP.large_footprint_raster(fs.n_visible, fs.n_pairs), (fs.n_visible, fs.n_pairs)
                one = VS.target(v, "f32", False)
                VS.ok(p, sc.ex(v, one, "f32", NO_CHUNKS, None if depths is None else depths[i]))
                assert p.frame_stats().rounds == 1 and one.tobytes() == host[i].tobytes(), ("raster2", i)
            for i, v in enumerate(vs):
                rounds = VS.target(v, "f32", False)
                VS.ok(p, sc.ex(v, rounds, "f32", CHUNKS, None if depths is None else depths[i]))
                assert p.frame_stats().rounds > 1 and rounds.tobytes() == host[i].tobytes(), ("rounds", i)
    finally:
        p.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# C: multi-sub-tile binning

@gpu
def test_c_multi_subtile_binning():
    _h100()
    vs = VS.multi_subtile_views()
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = VS.Scene(p, [(VS.room_cloud(VS.C_N, 13), "f32", None, B.CloudSettings())])
        for queued in (False, True):
            flags = ASYNC if queued else 0
            got, _ = _full_check(p, sc, vs, [("f32", False, flags), ("u8", True, flags)], None, (4, 6) if not queued else ())
            n_vis = got["stats"].n_visible
            assert KP.bin_multi_subtile(n_vis, KP.views_bin_grid(KP.H100_SMS, queued)), n_vis
    finally:
        p.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# D / E: multi-chunk key-gen over the view segments, many views

@gpu
@pytest.mark.parametrize("shape", ["64x1", "8x8"])
def test_d_multi_chunk_keygen(shape):
    _h100()
    p = B.GaussianSplattingPlugin(0)
    try:
        if shape == "64x1":
            cloud = VS.room_cloud(VS.D_N, 12)
            vs = VS.many_views(64)
            sc = VS.Scene(p, [(cloud, "f32", None, B.CloudSettings())])
            oracle_views = (0, 1, 2, 5)
        else:
            cloud = VS.room_cloud(VS.D_N8, 14)
            vs = VS.multi_subtile_views()
            sc = VS.Scene(p, VS.eight_entities(cloud))
            oracle_views = (6,)
        # (synchronous first: a queued first frame of a fresh context overflows its pair list and is not rendered)
        got, _ = _full_check(p, sc, vs, [("u8", True, 0), ("f32", False, ASYNC)], None, oracle_views)
        assert got["stats"].n == len(vs) * sc.n_view
        assert KP.keygen_multi_chunk(got["stats"].n, KP.scene_keygen_grid(queued=True))
        if shape == "64x1":
            nv = [int(((got["ids"] >= i * sc.n_view) & (got["ids"] < (i + 1) * sc.n_view)).sum()) for i in range(len(vs))]
            assert nv[5] == 0 and all(x > 0 for j, x in enumerate(nv) if j != 5), nv
    finally:
        p.destroy()


@gpu
def test_e_32_views_2_entities():
    _h100()
    vs = VS.many_views(32)
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = VS.Scene(p, VS.mixed_entities(VS.room_cloud(8000, 15)))
        depths = [VS.depth_buffer(v, 80 + i) for i, v in enumerate(vs)]
        got, _ = _full_check(p, sc, vs, [("f32", False, 0), ("u8", True, 0), ("f32", True, ASYNC)], depths, (0, 1, 2, 3))
        assert got["stats"].tiles_x == KP.views_tiles([(v.width, v.height) for v in vs])[-1]
        # the aux frame of the same views
        _full_check(p, sc, vs, [("f32", False, 0), ("u8", True, 0)], depths, (), aux=True)
    finally:
        p.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# F: starved grids

def _starve(p):
    h = p.add_cloud(VS.starve_cloud())
    p.render_view(h, B.CloudSettings(binning_rounds=False), VS.STARVE_VIEW, to_host=False)
    assert p.frame_stats().n_visible == 1
    h.destroy()


@gpu
@pytest.mark.parametrize("aux", [False, True])
def test_f_starved_grids(aux):
    """fresh (a new context), starved (after a frame of one visible entry: hint 1025) and hinted (the same frame again):
    every hook and pixel byte for byte; the starved frame's projection, splat depths and per-view range stride."""
    _h100()
    vs = VS.stride_views()
    cloud = VS.room_cloud(VS.F_N, 16)
    listed = VS.mixed_entities(cloud)
    if aux:
        listed[1] = (listed[1][0], listed[1][1], listed[1][2], B.CloudSettings(aabb=True, rasterize_mode=M.Depth))

    def frame(p, sc, depths):
        outs = _views(p, sc, vs, "f32", False, 0, depths, aux)
        h = VS.hooks(p, True)
        got = {k: (bytes(x) if k == "stats" else x.tobytes()) for k, x in h.items()}
        got["images"] = b"".join(o.tobytes() for trio in outs for o in (trio if aux else [trio]))
        return got, h

    p, q = B.GaussianSplattingPlugin(0), B.GaussianSplattingPlugin(0)
    try:
        sp, sq = VS.Scene(p, listed), VS.Scene(q, listed)
        depths = [VS.depth_buffer(v, 90 + i) for i, v in enumerate(vs)]
        fresh, _ = frame(p, sp, depths)
        _starve(q)
        starved, h = frame(q, sq, depths)
        hinted, _ = frame(q, sq, depths)
        for key in fresh:
            assert starved[key] == fresh[key], f"starved: {key} differs from the fresh frame's"
            assert hinted[key] == fresh[key], f"hinted: {key} differs from the fresh frame's"
        n_vis = h["stats"].n_visible
        hint = KP.projection_hint(1, h["stats"].n)
        assert hint == 1025
        assert KP.project_min_passes(n_vis, KP.project_grid(hint)) > 1, n_vis
        assert KP.splat_depth_passes(n_vis, KP.splat_depth_grid(hint)) > 1
        if aux:
            assert KP.depth_range_views_passes(n_vis, KP.depth_range_views_grid(hint)) > 1
        # the starved frame against the per-view frames and the oracle
        wants = _per_view(q, sq, vs, _views(q, sq, vs, "f32", False, 0, depths, aux), "f32", False, NO_CHUNKS, depths, aux)
        VS.check_restricted(h, wants, vs)
        if not aux:
            out = VS.target(vs[0], "f32", False)
            VS.ok(q, sq.ex(vs[0], out, "f32", NO_CHUNKS, depths[0]))
            VS.check_oracle(VS.hooks(q, True), out, sq.oracle_frame(vs[0], depths[0]))
    finally:
        q.destroy()
        p.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# G: the per-view Depth range at scale

@gpu
@pytest.mark.parametrize("with_colour", [False, True])
def test_g_depth_range_at_scale(with_colour):
    _h100()
    views = VS.depth_range_views()
    names, vs = list(views), list(views.values())
    cloud = VS.depth_range_cloud()
    listed = [(cloud, "f32", None, B.CloudSettings(rasterize_mode=M.Depth))]
    if with_colour:
        listed.append((cloud, "f32", VS.SC.transform((0.05, 0.0, 0.0)), B.CloudSettings(aabb=True)))
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = VS.Scene(p, listed)
        got, _ = _full_check(p, sc, vs, [("f32", False, 0), ("u8", True, 0)], None, (0, 3), aux=True)
        n, nvt = sc.n_view, got["stats"].n_visible
        srt = got["sorted"]
        counts = {}
        for i, name in enumerate(names):
            run = VS.visible_run(srt, nvt, i, n)
            counts[name] = len(run)
            lo, hi = VS.first_misses(run, n)
            if name.startswith("near0") or name == "near1":
                assert len(run) > 32 * 32 and lo >= 1024 and hi >= 1024, (name, lo, hi)
                assert KP.warp_first_miss_rounds(len(run), lo) > 1 and KP.warp_first_miss_rounds(len(run), hi) > 1
        k = len(listed)
        assert counts["all"] == n and counts["one"] == k and counts["none"] == 0 and counts["two"] == 2 * k, counts
        grid = KP.depth_range_views_grid(got["stats"].n)   # (a fresh context: the hint is N)
        assert KP.depth_range_views_passes(nvt, grid) == 1
        if k == 1:   # "two": its first two sorted positions in different CTAs of depth_range_views_kernel's grid
            i2 = names.index("two")
            pos = np.nonzero((srt[:nvt, 1] >= i2 * n) & (srt[:nvt, 1] < (i2 + 1) * n))[0]
            assert KP.depth_range_views_cta(int(pos[0]), grid) != KP.depth_range_views_cta(int(pos[1]), grid), pos
        # the single-view Depth frames agree with the oracle (the Depth colours over each view's own range)
        for i in (1, 4):
            out = VS.target(vs[i], "f32", False)
            VS.ok(p, sc.ex(vs[i], out, "f32", NO_CHUNKS))
            VS.check_oracle(VS.hooks(p, False), out, sc.oracle_frame(vs[i]))
    finally:
        p.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# H: the pair-list overflow at scale

@gpu
@pytest.mark.parametrize("queued", [False, True])
def test_h_pair_list_overflow(queued):
    _h100()
    vs = [B.perspective_view((x, 1.5, 3.0), (x, 1.5, -1.0), 960, 540) for x in (-0.032, 0.032)]
    p = B.GaussianSplattingPlugin(0)
    try:
        listed, bits, frame_box = V.entities("mixed")
        listed = [(c, layout, tr, dataclasses.replace(st, global_scale=6.0)) for c, layout, tr, st in listed]
        sc = VS.Scene(p, listed, bits, frame_box)
        outs = [VS.target(v, "f32", False) for v in vs]
        if queued:
            VS.ok(p, sc.views(vs, outs, "f32", ASYNC))
            assert p._lib.bgs_sync(p._ctx) == abi.BGS_NOT_READY
            VS.ok(p, sc.views(vs, outs, "f32", ASYNC))
            assert p.sync()
        else:
            VS.ok(p, sc.views(vs, outs, "f32"))
        got = VS.hooks(p, False)
        assert got["stats"].n_pairs > max(got["stats"].n, 1 << 20), got["stats"].n_pairs
        wants = _per_view(p, sc, vs, outs, "f32", False, NO_CHUNKS)
        VS.check_restricted(got, wants, vs)
        orc = sc.oracle_frame(vs[0])
        VS.check_oracle(wants[0], outs[0], orc)
    finally:
        p.destroy()
