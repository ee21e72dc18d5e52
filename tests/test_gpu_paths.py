"""Kernel paths that only queued, large or hinted frames reach, against the CPU oracle.

Which code a frame runs is picked from its size, the previous frame's counts, whether it is queued (BGS_FLAG_ASYNC) and
how far the context's buffers have grown; the results must not depend on it.  Every GPU case here renders in a fresh
context (so earlier tests' buffer growth does not decide what runs) and asserts, through `kernel_paths` (a restatement
of the library's selection rules), that it reached the path it exists for.  The bars are those of test_gpu_parity.py:
sorted entries, tile ranges, per-tile slices and projected geometry bit-exact, pixels within 1e-3.

Tests without the gpu mark check the selection table and that each input construction has the shape it is built for."""
import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import kernel_paths as KP
from test_gpu_parity import PIXEL_TOL, check_against_oracle, render_frame

gpu = pytest.mark.gpu
CAM = np.array([0.0, 1.5, 5.0], np.float32)          # headless_view's eye; it looks down -Z


# ---------------------------------------------------------------------------------------------------------------------
# the selection table (no GPU)

def test_radix_sort_path_table():
    P = KP.radix_sort_path
    # the benchmark's depth sort (C3: 721 340 visible of 6 M), hinted: one wave of 132 CTAs, 12 items
    assert P(721_340, 6_000_000) == (12, False, 132, 1)
    # a 6 M SORT_ALL sort: 3 waves of 264 CTAs, 16 items, peer-mask ranking
    assert P(6_000_000, 6_000_000) == (16, False, 264, 3)
    assert KP.depth_sort_path(6_000_000, 721_340, sort_all=True) == (16, False, 264, 3)
    assert KP.depth_sort_path(6_000_000, 721_340, sort_all=False) == (12, False, 132, 1)
    assert KP.depth_sort_path(6_000_000, 0, sort_all=False) == (16, False, 264, 3)          # no hint yet: n
    # more than 3 waves: MATCH.ANY
    assert P(6_500_000, 6_500_000).match_any and not P(6_200_000, 6_200_000).match_any
    # queued pair sorts run one CTA per SM: 3 waves end near 3.1 M
    assert KP.pair_sort_path(3_100_000, 4_000_000, queued=True) == (16, False, 132, 3)
    assert KP.pair_sort_path(3_300_000, 4_200_000, queued=True) == (16, True, 132, 4)
    assert KP.pair_sort_path(3_300_000, 4_200_000, queued=False) == (16, False, 264, 2)
    # the first queued frame of a fresh context plans for the whole pair buffer (max(2^20, n))
    assert KP.pair_sort_path(0, KP.initial_pair_capacity(6_000_000), queued=True).match_any
    # capacity floors the items: a buffer grown to 30 M pairs forces 15-16 items even for a small hint
    assert P(300_000, 1 << 20).items == 6
    assert P(300_000, 30_000_000).items == 16 and P(300_000, 30_000_000).waves == 1
    assert P(300_000, 62_500_000) == (16, False, 132, 1)
    assert KP.radix_status_rows(62_500_000) == 62_500_000 // 8192 + 1
    # tiny sorts
    assert P(0, 1 << 20) == (2, False, 132, 1) and P(1000, 1000) == (2, False, 132, 1)


def test_other_selection_rules():
    assert KP.pair_passes(KP.num_tiles(1920, 1080)) == 2 and KP.num_tiles(1920, 1080) == 8160
    assert KP.num_tiles(4112, 4112) == 66049 and KP.pair_passes(66049) == 3
    assert KP.pair_passes(KP.num_tiles(4096, 4096)) == 2                      # 65536 tiles: still 16-bit ids
    assert KP.num_tiles(65535, 304) == 4096 * 19 and KP.num_tiles(1, 1) == 1 and KP.pair_passes(1) == 1
    # key-gen phase 2 goes past one chunk beyond 16 tiles of 2048 per CTA
    assert KP.keygen_multi_chunk(4_500_000, 132) and not KP.keygen_multi_chunk(4_300_000, 132)
    assert not KP.keygen_multi_chunk(6_000_000, 528) and KP.keygen_multi_chunk(6_000_000, 132)
    # binning: more than 2048 ranks per CTA
    assert KP.bin_multi_subtile(400_000, 132) and not KP.bin_multi_subtile(400_000, 396)
    assert not KP.bin_multi_subtile(270_336, 132) and KP.bin_multi_subtile(270_337, 132)
    assert [KP.large_split_parts(n, 132) for n in (1, 33, 34, 66, 67, 132, 133, 264, 265)] == [16, 16, 8, 8, 4, 4, 2, 2, 1]
    assert [KP.footprint_class(t) for t in (0, 1, 4, 5, 128, 129)] == ["none", "tiny", "tiny", "medium", "medium", "large"]
    assert KP.chunked(8160, flag=True) and not KP.chunked(66049, flag=True) and not KP.chunked(8160, raster_mode=1, flag=True)
    assert not KP.chunked(8160, aux=True, flag=True) and not KP.chunked(8160, flag=False)
    assert KP.chunked(8160, n_vis_hint=100_000, n_pairs_hint=1 << 24) and not KP.chunked(8160, n_vis_hint=1 << 20, n_pairs_hint=1 << 24)
    assert KP.large_footprint_raster(1000, 8000) and not KP.large_footprint_raster(1000, 7999) and not KP.large_footprint_raster(0, 5)


# ---------------------------------------------------------------------------------------------------------------------
# position-only clouds: identity rotation, one scale and opacity, black (zero SH: np.zeros leaves the pages unwritten, so
# clouds of millions stay cheap on the host)

def position_cloud(pos, scale=0.002, opacity=0.6):
    n = len(pos)
    return B.PlanarGaussian3d(pos, np.zeros((n, 48), np.float32), np.tile(np.array([1, 0, 0, 0], np.float32), (n, 1)),
                              np.tile(np.array([scale, scale, scale, opacity], np.float32), (n, 1)))


def _at(z, x=0.0, y=1.5):
    """Points on (or near) the view axis; culled ones get z > 5 (behind the camera)."""
    z = np.asarray(z, np.float32)
    p = np.empty((len(z), 4), np.float32)
    p[:, 0], p[:, 1], p[:, 2], p[:, 3] = x, y, z, 1.0
    return p


# ---------------------------------------------------------------------------------------------------------------------
# adversarial depth keys.  key = (0xFFFFFFFF - bits(|p - cam|^2)) >> (32 - depth_bits); on the view axis |p - cam|^2 is
# dz * dz, one rounding

KINDS = ("equal", "two_interleaved", "low_digit", "high_digit", "far_to_near")
BITS = (16, 24, 32)


def key_pattern(kind, bits):
    """The distinct z values of a construction (visible, on the view axis)."""
    shift = 32 - bits
    if kind == "equal":
        return np.array([0.0], np.float32)
    if kind == "two_interleaved":
        return np.array([0.0, -1.0], np.float32)
    if kind == "low_digit":
        # squared distances whose float bits differ only in the shifted key's lowest digit: bucket centres of one
        # 256-bucket window (rounding z moves d^2 by a few ulp, far less than a bucket unless shift == 0; the edges of
        # the window are left out so it never carries into the next digit)
        base = np.array([1.25 * 2.0 ** 20], np.float32).view(np.uint32)[0] & ~np.uint32((1 << (shift + 8)) - 1)
        t = (np.uint64(base) + np.arange(8, 248, dtype=np.uint64) * np.uint64(1 << shift) + np.uint64((1 << shift) >> 1)).astype(np.uint32)
        d2 = t.view(np.float32).astype(np.float64)
        return (5.0 - np.sqrt(d2)).astype(np.float32)
    if kind == "high_digit":
        # |d| = 5 * 2^a: d^2 = 25 * 4^a, exact, so only the exponent bits 24..30 change (bit 23 keeps its parity)
        return (5.0 - 5.0 * 2.0 ** np.arange(-5, 21)).astype(np.float32)
    if kind == "far_to_near":
        return np.linspace(-3000.0, 4.5, 50_000).astype(np.float32)
    raise ValueError(kind)


def adversarial_z(kind, bits, n_vis, seed=0):
    pat = key_pattern(kind, bits)
    if kind in ("equal", "two_interleaved"):
        return pat[np.arange(n_vis) % len(pat)]
    if kind == "far_to_near":
        return pat[(np.arange(n_vis, dtype=np.int64) * len(pat)) // max(n_vis, 1)]   # index order: far to near
    return pat[np.random.default_rng(seed).integers(0, len(pat), n_vis)]


def build_positions(kind, bits, n_vis, n_culled, seed=0):
    """n_vis visible points of a construction with n_culled culled ones spread evenly between them."""
    n = n_vis + n_culled
    z = np.full(n, 10.0, np.float32)
    vis_idx = np.sort(np.random.default_rng(seed + 1).choice(n, n_vis, replace=False)) if n_culled else np.arange(n)
    z[vis_idx] = adversarial_z(kind, bits, n_vis, seed)
    return _at(z)


def _oracle_keys(oracle, pos, bits):
    return oracle.keygen(pos, B.headless_view(64, 64).to_abi(), B.GaussianSplattingPlugin.cloud_uniform(B.CloudSettings()), bits)


@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("kind", KINDS)
def test_adversarial_keys_have_their_shape(oracle, kind, bits):
    pos = build_positions(kind, bits, 20_000, 5_000, seed=3)
    keys = _oracle_keys(oracle, pos, bits)
    culled = np.uint32(0xFFFFFFFF >> (32 - bits))
    z_vis = pos[:, 2] < 5.0
    assert np.array_equal(keys == culled, ~z_vis), "the visible set must be exactly the constructed one"
    k = keys[z_vis].astype(np.int64)
    digits = [(k >> (8 * d)) & 255 for d in range(bits // 8)]
    distinct = [len(np.unique(x)) for x in digits]
    if kind == "equal":
        assert len(np.unique(k)) == 1
    elif kind == "two_interleaved":
        assert len(np.unique(k)) == 2 and np.all(k[0::2] == k[0]) and np.all(k[1::2] == k[1]) and k[0] != k[1]
    elif kind == "low_digit":
        # (32-bit keys: squares of adjacent f32 distances are ~2.5 ulp apart, so about 100 of the 240 targets are hit)
        assert distinct[0] >= (64 if bits == 32 else 200) and all(d == 1 for d in distinct[1:])
    elif kind == "high_digit":
        assert distinct[-1] >= 20 and all(d == 1 for d in distinct[:-1])
    else:
        assert np.all(np.diff(k) >= 0) and len(np.unique(k)) > 1000         # already in key order


# the depth sort's (items, grid, waves) combinations on this GPU class, and a hint that reaches each one
def depth_sort_combos(sm=KP.H100_SMS):
    """Every path launch_radix_sort can take for a synchronous-width sort, with the centre of the hint interval that
    reaches it (capacity = hint: what a SORT_ALL frame of that many gaussians runs)."""
    found = {}
    for h in range(1024, 7_000_000, 2048):
        found.setdefault(KP.radix_sort_path(h, h, sm), []).append(h)
    return {p: hs[len(hs) // 2] for p, hs in found.items()}


def sort_cases(sm=KP.H100_SMS):
    """-> (kind, bits, sort_all, hint, rel, expected SortPath).  SORT_ALL: one mostly-culled cloud per combination (its
    size is the hint), and the MATCH.ANY combination for every construction.  Compacted: every construction at every
    width, primed with a frame of `hint` visible gaussians, the target's visible count derived from the hint."""
    combos = sorted(depth_sort_combos(sm).items(), key=lambda kv: kv[1])
    raw = []
    for i, (path, hint) in enumerate(combos):
        raw.append((KINDS[i % 5], BITS[(i // 5) % 3], True, hint, "n"))
    match_hint = next(h for p, h in combos if p.match_any)
    for i, kind in enumerate(k for k in KINDS if k != raw[-1][0]):
        raw.append((kind, BITS[i % 3], True, match_hint, "n"))
    small = [h for p, h in combos if h <= 2_200_000]
    rels = ("equal", "tile+1", "tile-1", "x4", "quarter")
    for j, (kind, bits) in enumerate((k, b) for b in BITS for k in KINDS):
        h = small[(3 * j) % len(small)]
        rel = rels[j % len(rels)]
        if rel == "x4" and h > 1_000_000:
            rel = "quarter"
        raw.append((kind, bits, False, h, rel))
    cases = []
    for kind, bits, sort_all, hint, rel in raw:
        n, _, status_n = case_sizes(sort_all, hint, rel, sm)
        cases.append((kind, bits, sort_all, hint, rel, KP.depth_sort_path(n, hint, sort_all, sm, status_n)))
    return cases


def target_visible(hint, rel, sm=KP.H100_SMS):
    if rel in ("equal", "n"):
        return hint
    if rel == "x4":
        return 4 * hint
    if rel == "quarter":
        return max(1, hint // 4)
    tile = KP.RS_THREADS * KP.radix_sort_path(hint, hint, sm).items
    k = max(1, round(hint / tile))
    return k * tile + (1 if rel == "tile+1" else -1)


def case_sizes(sort_all, hint, rel, sm=KP.H100_SMS):
    """-> (cloud size, visible count, the status rows' capacity) of a sort case's target frame."""
    if sort_all:
        return hint, min(hint, 1_000_000), hint
    nv = target_visible(hint, rel, sm)
    n = nv + nv // 8
    return n, nv, max(n, hint)


SORT_CASES = sort_cases()


def test_sort_cases_cover_every_path():
    combos = set(depth_sort_combos())
    assert len(combos) == 16 and sum(p.match_any for p in combos) == 1
    reached = {want for *_, want in SORT_CASES}
    assert combos <= reached, combos - reached
    assert {(k, b, s) for k, b, s, *_ in SORT_CASES} == {(k, b, s) for k in KINDS for b in BITS for s in (False, True)}
    assert {r for *_, r, _ in SORT_CASES if r != "n"} == {"equal", "tile+1", "tile-1", "x4", "quarter"}
    assert {k for k, *_, want in SORT_CASES if want.match_any} == set(KINDS)


@gpu
@pytest.mark.parametrize("kind,bits,sort_all,hint,rel,want", SORT_CASES)
def test_depth_sort_variants_adversarial_keys(oracle, kind, bits, sort_all, hint, rel, want):
    sm = KP.device_sm_count()
    n, n_vis, status_n = case_sizes(sort_all, hint, rel, sm)
    # (the table was built for 132 SMs: on another device the same frames take other paths)
    assert KP.depth_sort_path(n, hint, sort_all, sm, status_n) == want, f"{sm} SMs: this case no longer reaches {want}"
    view = B.headless_view(40, 40)           # the view axis crosses the middle of tile (1, 1)
    s = B.CloudSettings(radix_sort_depth_bits=B.RadixSortDepthBits(bits), sort_all=sort_all)
    p = B.GaussianSplattingPlugin(0)
    try:
        if not sort_all:
            prime = p.add_cloud(position_cloud(_at(np.zeros(hint, np.float32))))
            p.render_view(prime, s, view, to_host=False)
            assert p.frame_stats().n_visible == hint
            prime.destroy()
        pos = build_positions(kind, bits, n_vis, n - n_vis, seed=bits)
        h = p.add_cloud(position_cloud(pos))
        p.render_view(h, s, view, to_host=False)
        assert p.frame_stats().n_visible == n_vis
        keys = _oracle_keys(oracle, pos, bits)
        sk, si = oracle.radix_sort(keys, bits)
        got = p.sorted_entries()
        assert np.array_equal(got[:, 0], sk), f"sorted keys differ on {want}"
        assert np.array_equal(got[:, 1], si), f"sort permutation differs on {want}"
        h.destroy()
    finally:
        p.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# queued frames at size

@gpu
def test_queued_c3_frame_vs_oracle(oracle):
    """The configuration bench.py times: C3 (6 M f16 gaussians, 1080p) queued.  Its first frame in a fresh context runs
    the MATCH.ANY pair sort (planned for the whole 6 M pair buffer), the multi-chunk key-gen and the multi-sub-tile
    binning; the hinted second frame runs the 12-item one-wave depth sort."""
    sm = KP.device_sm_count()
    cloud = B.random_gaussians_3d_seeded(6_000_000, 0)
    p = B.GaussianSplattingPlugin(0)
    try:
        n = len(cloud)
        assert KP.keygen_multi_chunk(n, KP.coop_grid(sm, 1, queued=True))
        _, til = check_against_oracle(p, oracle, cloud, B.CloudSettings(global_scale=0.02), B.headless_view(1920, 1080),
                                      f16=True, asynchronous=True)
        nv, npairs = til["n_vis"], til["n_pairs"]
        assert KP.bin_multi_subtile(nv, KP.coop_grid(sm, 1, queued=True))
        assert KP.pair_sort_path(0, KP.initial_pair_capacity(n), queued=True, sm_count=sm).match_any
        assert npairs <= KP.initial_pair_capacity(n)
        assert KP.depth_sort_path(n, 0, False, sm) == (16, False, 2 * sm, 3)
        assert KP.depth_sort_path(n, nv, False, sm).waves == 1
        assert KP.pair_sort_path(npairs, KP.initial_pair_capacity(n), queued=True, sm_count=sm).waves > 1
    finally:
        p.destroy()


@gpu
def test_queued_keygen_multi_chunk_mostly_behind_camera(oracle):
    """4.5 M gaussians, 1 in 61 in front of the camera and spread over every key-gen CTA's range: queued frames have
    132 key-gen CTAs, so each expands 17 tiles of mask words in two chunks."""
    sm = KP.device_sm_count()
    n = 4_500_000
    cloud = B.random_gaussians_3d_seeded(n, 7)
    pos = cloud.position_visibility
    behind = np.ones(n, bool); behind[::61] = False
    pos[behind, 2] = np.abs(pos[behind, 2]) + 5.5
    # the others inside the frustum (headless_view: half-height 0.41, half-width 0.74 per unit of distance)
    rng = np.random.default_rng(7)
    m = int((~behind).sum())
    dist = rng.uniform(2.0, 20.0, m).astype(np.float32)
    pos[~behind, 0] = rng.uniform(-0.6, 0.6, m).astype(np.float32) * dist
    pos[~behind, 1] = np.float32(1.5) + rng.uniform(-0.35, 0.35, m).astype(np.float32) * dist
    pos[~behind, 2] = np.float32(5.0) - dist
    assert KP.keygen_multi_chunk(n, KP.coop_grid(sm, 1, queued=True))
    view = B.headless_view(960, 540)
    s = B.CloudSettings(global_scale=0.02)
    p = B.GaussianSplattingPlugin(0)
    try:
        _, til = check_against_oracle(p, oracle, cloud, s, view, asynchronous=True)
        assert til["n_vis"] > 60_000
        # the visible ones sit in every CTA's second chunk too
        tiles = -(-n // KP.KG_TILE)
        keys = oracle.keygen(pos, view.to_abi(), p.cloud_uniform(s), 32)
        vis_idx = np.flatnonzero(keys != 0xFFFFFFFF)
        assert len(vis_idx) == til["n_vis"]
        second = [(b * tiles // sm) * KP.KG_TILE + KP.KG_CHUNK_TILES * KP.KG_TILE for b in range(sm)
                  if ((b + 1) * tiles // sm - b * tiles // sm) > KP.KG_CHUNK_TILES]
        assert len(second) > sm // 2
        assert all(np.any((vis_idx >= s) & (vis_idx < s + KP.KG_TILE)) for s in second)
    finally:
        p.destroy()


@gpu
@pytest.mark.parametrize("asynchronous", [True, False])
def test_binning_multi_subtile(oracle, asynchronous):
    """About 400 k visible splats: queued frames bin them with 132 CTAs, more than 2048 ranks each (`!single`)."""
    sm = KP.device_sm_count()
    cloud = B.random_gaussians_3d_seeded(3_400_000, 12)
    p = B.GaussianSplattingPlugin(0)
    try:
        _, til = check_against_oracle(p, oracle, cloud, B.CloudSettings(global_scale=0.01), B.headless_view(1280, 720),
                                      asynchronous=asynchronous)
        assert 350_000 < til["n_vis"] < 450_000
        if asynchronous:
            assert KP.bin_multi_subtile(til["n_vis"], KP.coop_grid(sm, 1, queued=True))
    finally:
        p.destroy()


@gpu
def test_three_queued_views_each_vs_its_oracle_frame(oracle):
    """Three queued frames with different views back to back, each delivered to its own host array: every one must be
    its own view's frame (the library alternates two device frames and copies out on a second stream)."""
    cloud = B.random_gaussians_3d_seeded(300_000, 21)
    s = B.CloudSettings(global_scale=0.05)
    views = [B.orbit_view(i, 3, 640, 360) for i in range(3)]
    p = B.GaussianSplattingPlugin(0)
    h = p.add_cloud(cloud)
    try:
        for _ in range(3):     # (the first pass may grow the pair buffer)
            outs = [np.full((360, 640, 4), np.nan, np.float32) for _ in views]
            for v, o in zip(views, outs):
                p.render_view(h, s, v, fmt="rgba32f", out=o, asynchronous=True)
            if p.sync():
                break
        else:
            raise AssertionError("queued frames kept outgrowing the pair buffer")
        u = p.cloud_uniform(s, None, h.aabb)
        for v, o in zip(views, outs):
            til = oracle.render_tiles(cloud, v.to_abi(), u, s.to_abi())
            assert float(np.abs(o - til["image"]).max()) <= PIXEL_TOL
        # the hooks describe the last frame
        assert p.frame_stats().n_visible == til["n_vis"] and np.array_equal(p.tile_ranges(), til["tile_ranges"])
        assert np.array_equal(p.tile_entries(), til["tile_entries"])
        assert not np.array_equal(outs[0], outs[1]) and not np.array_equal(outs[1], outs[2])
    finally:
        h.destroy()
        p.destroy()


@gpu
def test_queued_pair_sort_match_any(oracle):
    """A queued frame with more than 3.2 M pairs after a synchronous frame of that size set the hint: one CTA per SM
    needs more than 3 waves, so the pair sort runs MATCH.ANY ranking.  Pair-list bars against the oracle."""
    sm = KP.device_sm_count()
    n = 2_000_000
    cloud = B.random_gaussians_3d_seeded(n, 5)
    view = B.headless_view(1920, 1080)
    s = B.CloudSettings(global_scale=0.12, binning_rounds=False)
    p = B.GaussianSplattingPlugin(0)
    h = p.add_cloud(cloud)
    try:
        p.render_view(h, s, view, to_host=False)
        fs = p.frame_stats()
        npairs = fs.n_pairs
        cap = KP.grown_pair_capacity(KP.initial_pair_capacity(n), npairs)
        path = KP.pair_sort_path(npairs, cap, queued=True, sm_count=sm)
        assert path.match_any, (npairs, path)
        img = render_frame(p, h, s, view, asynchronous=True)
        u = p.cloud_uniform(s, None, h.aabb)
        til = oracle.render_tiles(cloud, view.to_abi(), u, s.to_abi())
        assert p.frame_stats().n_pairs == til["n_pairs"] == npairs
        assert np.array_equal(p.tile_ranges(), til["tile_ranges"])
        assert np.array_equal(p.tile_entries(), til["tile_entries"])
        assert float(np.abs(img - til["image"]).max()) <= PIXEL_TOL
    finally:
        h.destroy()
        p.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# tile-grid edges

EDGE_VIEWS = [(4112, 4112), (65535, 304), (304, 65535), (1, 1), (16, 16), (17, 1)]


@gpu
@pytest.mark.parametrize("w,h", EDGE_VIEWS)
def test_tile_grid_edges(oracle, w, h):
    tiles = KP.num_tiles(w, h)
    cloud = B.random_gaussians_3d_seeded(20_000, 31)
    s = B.CloudSettings(global_scale=0.3 if max(w, h) < 100 else 0.05)
    p = B.GaussianSplattingPlugin(0)
    try:
        img, til = check_against_oracle(p, oracle, cloud, s, B.headless_view(w, h))
        assert til["n_vis"] > 0 and til["n_pairs"] > 0
        h2 = p.add_cloud(cloud)
        try:
            assert np.array_equal(p.render_view(h2, s, B.headless_view(w, h)), img)
            fs = p.frame_stats()
            assert fs.tiles_x * fs.tiles_y == tiles and fs.rounds == 1 and fs.n_pairs == til["n_pairs"]
            if (w, h) == (4112, 4112):
                assert KP.pair_passes(tiles) == 3
                assert int(til["tile_ranges"][65536:, 1].max()) > 0, "tile ids >= 2^16 must hold pairs"
                # more than 65 536 tiles: never binned in rounds, whatever the flag says
                assert not KP.chunked(tiles, flag=True)
                forced = p.render_view(h2, B.CloudSettings(global_scale=0.05, binning_rounds=True), B.headless_view(w, h))
                assert p.frame_stats().rounds == 1 and np.array_equal(forced, img)
                # the largest chunkable frame in the same context: its five per-round range arrays (5 x 65 536 entries)
                # and 65 536 done bytes must fit the arena the 66 049-tile frame left behind (api.cu ensure_arena), which a
                # one-round sizing (66 049 entries) would not
                v2 = B.headless_view(4096, 4096)
                t2 = KP.num_tiles(4096, 4096)
                assert t2 == KP.CHUNK_MAX_TILES and KP.chunked(t2, flag=True) and 5 * t2 > tiles
                s_one = B.CloudSettings(global_scale=0.05, binning_rounds=False)
                s_many = B.CloudSettings(global_scale=0.05, binning_rounds=True)
                many = p.render_view(h2, s_many, v2)
                assert p.frame_stats().rounds == 5 and p.frame_stats().tiles_x * p.frame_stats().tiles_y == t2
                one = p.render_view(h2, s_one, v2)
                assert p.frame_stats().rounds == 1
                assert np.array_equal(one, many)
                til2 = oracle.render_tiles(cloud, v2.to_abi(), p.cloud_uniform(s_one, None, h2.aabb), s_one.to_abi())
                assert float(np.abs(one - til2["image"]).max()) <= PIXEL_TOL
        finally:
            h2.destroy()
    finally:
        p.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# raster chunk edges: exactly K splats on the frame's last tile, around the 256-entry chunks the blend streams through
# its bulk-copy double buffer

RASTER_W, RASTER_H = 31, 16                      # two tiles; odd width: tile 1 is 15 pixels wide
RASTER_KS = (1, 255, 256, 257, 512, 513, 1025)
RASTER_OPACITY = {"low": 0.002, "mid": 0.12, "high": 0.6}   # never saturates / in chunk 1 / in chunk 0
RASTER_SETTINGS = dict(opacity_adaptive_radius=False)        # (the adaptive radius would shrink the faint splats to nothing)


def raster_edge_cloud(k, lead, opacity, seed=0):
    """K large splats centred on tile 1 (each covers all of it and reaches into tile 0) behind `c` small ones that only
    touch tile 0, with c chosen so tile 1's slice starts at (c + K) % 4 == lead.  Tile 1 is the last tile: its slice ends
    at the end of the pair list.  Depths are shuffled against index order."""
    c = (lead - k) % 4
    rng = np.random.default_rng(seed)
    view = B.headless_view(RASTER_W, RASTER_H)
    t, aspect = np.tan(np.pi / 8), RASTER_W / RASTER_H
    def at(px, py, d):
        ndc_x, ndc_y = (px - RASTER_W / 2) / (RASTER_W / 2), (RASTER_H / 2 - py) / (RASTER_H / 2)
        return np.stack([ndc_x * d * t * aspect, 1.5 + ndc_y * d * t, 5.0 - d, np.ones_like(d)], 1)
    d_big = rng.uniform(4.0, 6.0, k)
    d_small = rng.uniform(2.0, 3.0, c)
    pos = np.concatenate([at(23.5, 8.0, d_big), at(5.0, 8.0, d_small)]).astype(np.float32)
    n = len(pos)
    so = np.empty((n, 4), np.float32)
    so[:k, :3] = (0.45 * d_big)[:, None]          # ~7 px sigma at any depth
    so[k:, :3] = 0.004
    so[:, 3] = opacity
    sh = rng.uniform(-1, 1, (n, 48)).astype(np.float32)
    rot = np.tile(np.array([1, 0, 0, 0], np.float32), (n, 1))
    perm = rng.permutation(n)
    return B.PlanarGaussian3d(pos[perm], sh[perm], rot, so[perm]), view


RASTER_CASES = [(k, lead, op) for i, (k, op) in enumerate((k, op) for k in RASTER_KS for op in RASTER_OPACITY)
                for lead in ([i % 4] if k <= 256 else [i % 4, (i + 2) % 4])]


def test_raster_edge_cases_have_their_shape(oracle):
    leads = set()
    for k, lead, op in RASTER_CASES:
        cloud, view = raster_edge_cloud(k, lead, RASTER_OPACITY[op])
        s = B.CloudSettings(**RASTER_SETTINGS)
        til = oracle.render_tiles(cloud, view.to_abi(), B.GaussianSplattingPlugin.cloud_uniform(s), s.to_abi())
        r = til["tile_ranges"]
        assert r[1, 1] - r[1, 0] == k and r[1, 1] == til["n_pairs"], (k, lead, r)
        assert KP.raster_lead(int(r[1, 0])) == lead
        assert r[0, 1] - r[0, 0] == k + (lead - k) % 4
        if k > 256:
            leads.add(lead)
        layer = oracle.render_ref(cloud, view.to_abi(), B.GaussianSplattingPlugin.cloud_uniform(s), s.to_abi(),
                                  dst=np.zeros((RASTER_H, RASTER_W, 4), np.float32))
        coverage = layer[:, 16:, 3]                                    # 1 - T over tile 1
        if op == "low":
            assert coverage.max() < 1 - 1e-4 and coverage.min() > 0   # covered, never saturated
        elif op == "high" and k >= 256:
            assert coverage.min() >= 1 - 1e-4                         # the whole tile saturates (in chunk 0)
        elif op == "mid" and k >= 513:
            assert coverage.min() >= 1 - 1e-4
    assert leads == {0, 1, 2, 3}
    assert {k for k, *_ in RASTER_CASES} == set(RASTER_KS)


@gpu
@pytest.mark.parametrize("k,lead,op", RASTER_CASES)
def test_raster_chunk_edges_and_variants(oracle, k, lead, op):
    """The oracle bar on MODE 0's raster_kernel, then byte identity of every other blend of the same frame: binning rounds
    (raster2_kernel<true>), raster2_kernel<false> (picked after a frame of large footprints), and the colour frame of
    bgs_render_aux (MODE 0's aux raster_kernel), in all three formats and with premultiplied output.  USE_AABB frames
    (MODE 1 and 2) are checked against the oracle."""
    import dataclasses

    cloud, view = raster_edge_cloud(k, lead, RASTER_OPACITY[op])
    s = B.CloudSettings(binning_rounds=False, **RASTER_SETTINGS)
    p = B.GaussianSplattingPlugin(0)
    try:
        img, til = check_against_oracle(p, oracle, cloud, s, view)      # fresh context: MODE 0's raster_kernel, hinted frame too
        assert til["tile_ranges"][1, 1] - til["tile_ranges"][1, 0] == k
        h = p.add_cloud(cloud)
        heavy = p.add_cloud(B.random_gaussians_3d_seeded(200, 3))
        try:
            frames = {}
            for fmt in ("rgba32f", "rgba16f", "rgba8_srgb"):
                for premul in (False, True):
                    base = p.render_view(h, s, view, fmt=fmt, premultiplied=premul)
                    fs = p.frame_stats()
                    assert not KP.large_footprint_raster(fs.n_visible, fs.n_pairs)     # next frame: MODE 0's raster_kernel again
                    again = p.render_view(h, s, view, fmt=fmt, premultiplied=premul)
                    rounds = p.render_view(h, dataclasses.replace(s, binning_rounds=True), view, fmt=fmt, premultiplied=premul)
                    assert p.frame_stats().rounds == 5
                    p.render_view(heavy, B.CloudSettings(global_scale=2.0, binning_rounds=False), B.headless_view(512, 512), to_host=False)
                    fs = p.frame_stats()
                    assert KP.large_footprint_raster(fs.n_visible, fs.n_pairs)
                    r2 = p.render_view(h, s, view, fmt=fmt, premultiplied=premul)
                    for name, f in (("hinted", again), ("rounds", rounds), ("raster2", r2)):
                        assert np.array_equal(f.view(np.uint8), base.view(np.uint8)), (fmt, premul, name)
                    frames[(fmt, premul)] = base
            assert np.array_equal(frames[("rgba32f", False)], img)
            colour, _, _ = p.render_view_aux(h, s, view, fmt="rgba32f")
            assert np.array_equal(colour, img)
        finally:
            h.destroy()
            heavy.destroy()
        for gm in (B.GaussianMode.Gaussian3d, B.GaussianMode.Gaussian2d):
            check_against_oracle(p, oracle, cloud, B.CloudSettings(aabb=True, gaussian_mode=gm, **RASTER_SETTINGS), view)
    finally:
        p.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# every f16 opacity: the 65 536-entry adaptive-cutoff table (f16 clouds) and the in-kernel det_ln (f32 clouds)

def every_f16_opacity_cloud():
    """One gaussian per f16 bit pattern of the opacity (NaNs, infinities, negatives, subnormals included) on a 256 x 256
    grid across headless_view(512, 512); everything else fixed."""
    op = np.arange(65536, dtype=np.uint32).astype(np.uint16).view(np.float16).astype(np.float32)
    g = (np.arange(256, dtype=np.float32) - np.float32(127.5)) * np.float32(3.9 / 256)
    pos = np.stack([np.tile(g, 256), np.float32(1.5) + np.repeat(g, 256), np.zeros(65536, np.float32),
                    np.ones(65536, np.float32)], 1)
    cloud = position_cloud(pos, scale=0.004)
    cloud.scale_opacity[:, 3] = op
    cloud.spherical_harmonic[:, :3] = 0.8
    return cloud


def test_every_f16_opacity_survives_the_upload():
    cloud = every_f16_opacity_cloud()
    bits = cloud.pack_f16()[1][:, 3] & 0xFFFF
    assert np.array_equal(np.sort(bits), np.arange(65536)), "the f16 upload must carry every opacity bit pattern"
    assert np.array_equal(cloud.rounded_to_f16().scale_opacity[:, 3].view(np.uint32), cloud.scale_opacity[:, 3].view(np.uint32))


@gpu
@pytest.mark.parametrize("f16", [True, False])
def test_every_f16_opacity_vs_oracle(oracle, f16):
    """Geometry, bboxes (adaptive radius on) and colours bit-exact for every opacity value; pixels NaN exactly where the
    oracle's are and within the bar elsewhere."""
    cloud = every_f16_opacity_cloud()
    view = B.headless_view(512, 512)
    s = B.CloudSettings(opacity_adaptive_radius=True)
    p = B.GaussianSplattingPlugin(0)
    try:
        h = p.add_cloud(cloud, f16=f16)
        img = p.render_view(h, s, view, fmt="rgba32f")
        u = p.cloud_uniform(s, None, h.aabb)
        oc = cloud.rounded_to_f16() if f16 else cloud          # (the scale and colour planes are rounded too)
        til = oracle.render_tiles(oc, view.to_abi(), u, s.to_abi())
        assert p.frame_stats().n_visible == til["n_vis"] == 65536
        assert np.array_equal(p.tile_ranges(), til["tile_ranges"]) and np.array_equal(p.tile_entries(), til["tile_entries"])
        rec, ids = p.projected()
        assert np.array_equal(ids, til["rank_to_id"])
        orec = oracle.project(oc, view.to_abi(), u, s.to_abi(), til["rank_to_id"])
        drawn = orec["xlo"] <= orec["xhi"]
        assert 1000 < drawn.sum() < 65536                      # some opacities draw nothing, most draw something
        geo = np.stack([orec[k] for k in ("cx", "cy", "ux", "uy", "vx", "vy")], 1)
        assert np.array_equal(rec[drawn, :6].view(np.uint32), geo[drawn].view(np.uint32)), "projected geometry not bit-exact"
        bb = rec[:, 6:8].view(np.uint32)
        assert np.array_equal(bb[drawn, 0], orec["xlo"][drawn].astype(np.uint32) | (orec["xhi"][drawn].astype(np.uint32) << 16))
        assert np.array_equal(bb[drawn, 1], orec["ylo"][drawn].astype(np.uint32) | (orec["yhi"][drawn].astype(np.uint32) << 16))
        assert np.all((bb[~drawn, 0] & 0xFFFF) > (bb[~drawn, 0] >> 16))
        col = np.stack([orec[k] for k in ("r", "g", "b", "op")], 1)
        assert np.allclose(rec[drawn, 8:12], col[drawn], rtol=0, atol=1e-4, equal_nan=True)
        want = til["image"]
        nan = np.isnan(want)
        assert np.array_equal(np.isnan(img), nan), "NaN pixels differ from the oracle's"
        assert float(np.abs(img[~nan] - want[~nan]).max()) <= PIXEL_TOL
        h.destroy()
    finally:
        p.destroy()
