"""Tile binning's footprint classes, large-footprint splits and pair-count limits, against the CPU oracle.

bin_emit_coop_kernel (csrc/bin.cu) writes a splat's (tile, rank) pairs on one of three paths, picked by how many tiles
its bbox touches: tiny footprints (<= 4 tiles) by the thread that owns the rank, medium ones (5..128) from the front
of the queue arrays 32 splats per warp, large ones (> 128) from the back of the queue arrays, each cut into 1..16
32-aligned parts dealt round-robin over the grid's warps.  The inputs here are built splat by splat so that each one's
bbox covers an exact tile rectangle, which lets a test put footprints on the class boundaries, choose how many large
splats there are (and so the part count) and where the pair buffer's capacity falls.  `kernel_paths` restates the
rules, and every GPU case asserts that it reached the path it exists for on this device.

Each GPU case renders in a fresh context, after a decoy frame: a larger cloud on the same tile grid that leaves its
own pairs in the pair buffers and grows the cloud-sized buffers, so the large queue sits at the back of a buffer larger
than the frame needs.  A slot the kernel forgets to write then holds a stale pair (a valid tile id of this grid) and
shows up in the comparison.  n_visible, n_pairs, the rank order, the tile ranges and the per-tile entries must match
`render_tiles` bit for bit.

Tests without the gpu mark pin the rules' table and check that every construction has the shape it is built for."""
import dataclasses
import functools
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import kernel_paths as KP
from bevy_gaussian_splatting_b200 import abi
from test_gpu_parity import PIXEL_TOL, check_against_oracle, render_frame

gpu = pytest.mark.gpu

TILES = 130                                   # 130 x 130 tiles: a 129-tile row or column fits
VIEW = B.headless_view(16 * TILES, 16 * TILES)
S = B.CloudSettings(opacity_adaptive_radius=False, binning_rounds=False)   # cutoff 3 sigma whatever the opacity
S_ROUNDS = dataclasses.replace(S, binning_rounds=True)
UNIFORM = B.GaussianSplattingPlugin.cloud_uniform(S)
SM = KP.H100_SMS                              # the sizes below are chosen for this SM count; GPU tests assert it
MODES = [pytest.param(False, id="sync"), pytest.param(True, id="queued")]

NONE, LEFT, RIGHT, TOP, BOTTOM, COVER = range(6)   # where a splat's bbox is clipped by the frame
TINY_SIZES = [(1, 1), (1, 2), (2, 1), (1, 3), (3, 1), (2, 2), (1, 4), (4, 1)]
MEDIUM_SIZES = [(1, 5), (5, 1), (2, 3), (3, 2), (3, 3), (4, 4), (5, 7), (11, 11), (8, 16), (1, 128)]
LARGE_SIZES = [(1, 129), (129, 1), (3, 43), (43, 3), (27, 19), (19, 27), (32, 16), (16, 32), (15, 17), (7, 73),
               (73, 7), (2, 65), (31, 5), (32, 5), (33, 4), (64, 3), (65, 2), (130, 1), (130, 2), (33, 5)]
ROUND_FRACS = (16, 128, 1024, 8192)           # api.cu CHUNK_FRAC: the inner round boundaries, in 1/65536 of n_visible


# ---------------------------------------------------------------------------------------------------------------------
# the rules' table (no GPU)

def test_binning_rule_table():
    q, s = KP.bin_grid(SM, queued=True), KP.bin_grid(SM, queued=False)
    assert (q, s) == (132, 396) and (q * KP.BIN_WARPS_PER_CTA, s * KP.BIN_WARPS_PER_CTA) == (1056, 3168)
    for grid, ends in ((q, (33, 66, 132, 264)), (s, (99, 198, 396, 792))):
        for parts, hi in zip((16, 8, 4, 2), ends):
            assert KP.large_split_parts(hi, grid) == parts and KP.large_split_parts(hi + 1, grid) == parts // 2
        assert KP.large_split_parts(1, grid) == 16 and KP.large_split_parts(100_000, grid) == 1
    assert KP.medium_passes(33_792, q) == 1 and KP.medium_passes(33_793, q) == 2
    assert KP.medium_passes(101_376, s) == 1 and KP.medium_passes(101_377, s) == 2
    assert KP.medium_passes(20, q) == 1 and KP.medium_passes(0, s) == 0
    assert KP.large_tickets(1056, q) == (1, 1) and KP.large_tickets(1057, q) == (1, 2)
    assert KP.large_tickets(3168, s) == (1, 1) and KP.large_tickets(3169, s) == (1, 2)
    assert KP.large_tickets(33, q) == (16, 1) and KP.large_tickets(34, q) == (8, 1)
    # 300 000 ranks: 2272 or 2273 per queued CTA, two sub-tiles of up to 2048; one sub-tile per synchronous CTA
    assert KP.bin_subtiles(300_000, q)[0] == [(0, 2048), (2048, 2272)] and KP.bin_subtiles(300_000, q)[-1][-1][1] == 300_000
    assert all(len(x) == 1 for x in KP.bin_subtiles(300_000, s))
    # part slices: 129 tiles at 16 parts -> per = 32, part 4 is the single pair [128, 129), parts 5..15 empty
    sl = KP.large_part_slices(129, 16)
    assert sl[:5] == [(0, 32), (32, 64), (64, 96), (96, 128), (128, 129)] and all(a == b for a, b in sl[5:])
    sl = KP.large_part_slices(513, 16)
    assert sl[7] == (448, 512) and sl[8] == (512, 513) and all(a == b for a, b in sl[9:])
    assert KP.large_part_slices(512, 16)[-1] == (480, 512) and KP.large_part_slices(511, 16)[-1] == (480, 511)
    assert KP.large_part_slices(200, 1) == [(0, 200)]
    assert KP.footprint_rect(16, 31, 0, 15) == (1, 0, 1, 1) and KP.footprint_rect(15, 16, 17, 64) == (0, 1, 2, 4)
    assert KP.footprint_rect(1, 0, 1, 0) == (0, 0, 0, 0)


def _cuobjdump():
    found = shutil.which("cuobjdump")
    if found:
        return found
    return os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")


def test_bin_kernel_occupancy_matches_the_pinned_fit():
    """KP.BIN_CTAS_PER_SM_FIT against the built kernel's registers and shared memory, with sm_90's allocation rules:
    registers in units of 256 per warp out of 65 536, shared memory plus 1 KB per CTA out of 228 KB, 2048 threads
    and 32 CTAs per SM."""
    lib = abi.LIB_PATH
    if not os.path.exists(lib):
        pytest.skip("libbgs.so is not built")
    out = subprocess.run([_cuobjdump(), "--dump-resource-usage", lib], check=True, capture_output=True, text=True).stdout
    m = re.search(r"Function \S*bin_emit_coop_kernel\S*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", out)
    assert m, "bin_emit_coop_kernel not found in libbgs.so"
    regs, stack, shared, local = map(int, m.groups())
    threads = 256                                          # bin.cu:12 (BIN_THREADS)
    warp_regs = -(-regs * 32 // 256) * 256
    by_regs = (65536 // warp_regs) // (threads // 32)
    by_shared = (228 * 1024) // (shared + 1024)
    fit = min(by_regs, by_shared, 2048 // threads, 32)
    assert fit == KP.BIN_CTAS_PER_SM_FIT, (regs, shared, fit)
    assert stack == 0 and local == 0


# ---------------------------------------------------------------------------------------------------------------------
# splats built to exact footprints

def footprint_cloud(rects, seed=0, view=VIEW, opacity=0.35, d0=3.0, d1=25.0):
    """A cloud whose rank-r splat's oracle bbox covers exactly the tile rectangle rects[r] = (tx0, ty0, w, h, clip).

    Unclipped splats are centred on their rectangle and keep 4-5 px inside its edges.  LEFT/RIGHT/TOP/BOTTOM splats
    are centred near that frame edge and reach past it, so the rectangle (which starts at that edge) is what the clamp
    leaves; COVER splats reach past every edge.  Ranks follow the distance from the camera (d0 .. d1, rank order);
    the cloud's index order is shuffled.  Each splat is flat (tiny z scale) and facing the camera, so its screen
    covariance is its xy covariance scaled by the focal length over its depth; it is turned about the view axis by a
    small angle (an exactly diagonal covariance meets the eigenvector quirk of test_edge_cases), and its two scales
    solve for the wanted half-extents at that angle.  -> (cloud, idx): cloud index i holds rank idx[i]."""
    rects = np.asarray(rects, np.int64).reshape(-1, 5)
    n = len(rects)
    W, H = float(view.width), float(view.height)
    tx0, ty0, w, h, clip = (rects[:, k].astype(np.float64) for k in range(5))
    cx, hx = 16 * tx0 + 8 * w, 8 * w - 4
    cy, hy = 16 * ty0 + 8 * h, 8 * h - 5
    lx, ly = 16 * w - 4, 16 * h - 5
    for side, sel_x, at in ((LEFT, True, lambda L: 0.25 * L), (RIGHT, True, lambda L: W - 0.25 * L),
                            (TOP, False, lambda L: 0.25 * L), (BOTTOM, False, lambda L: H - 0.25 * L)):
        m = clip == side
        if sel_x:
            cx[m], hx[m] = at(lx[m]), 0.75 * lx[m]
        else:
            cy[m], hy[m] = at(ly[m]), 0.75 * ly[m]
    m = clip == COVER
    cx[m], hx[m], cy[m], hy[m] = W / 2, W / 2 + 40, H / 2, H / 2 + 45
    rng = np.random.default_rng(seed)
    theta = np.minimum(0.25 * np.minimum(hx, hy) / np.maximum(hx, hy), 0.05) * np.where(rng.random(n) < 0.5, -1.0, 1.0)
    c, s = np.cos(theta), np.abs(np.sin(theta))
    det = c * c - s * s
    ba, bb = 2 * (c * hx - s * hy) / det, 2 * (c * hy - s * hx) / det     # 3-sigma screen extents along the axes
    f = float(view.clip_from_view[1, 1])
    a, b = (cx - W / 2) / (f * H / 2), (H / 2 - cy) / (f * H / 2)
    dist = d0 + (d1 - d0) * np.arange(n) / max(n, 1)
    t = dist / np.sqrt(1 + a * a + b * b)                    # view depth
    sa = t / (f * H) * np.sqrt((ba / 3) ** 2 - 0.3)           # (the projection adds 0.3 px^2 of blur to each axis)
    sb = t / (f * H) * np.sqrt((bb / 3) ** 2 - 0.3)
    pos = np.stack([a * t, 1.5 + b * t, 5.0 - t, np.ones(n)], 1)
    rot = np.stack([np.cos(theta / 2), np.zeros(n), np.zeros(n), np.sin(theta / 2)], 1)
    so = np.stack([sa, sb, 1e-3 * np.minimum(sa, sb), np.full(n, opacity)], 1)
    sh = np.zeros((n, 48), np.float32)
    sh[:, :3] = rng.uniform(-0.8, 0.8, (n, 3))
    idx = rng.permutation(n)
    cloud = B.PlanarGaussian3d(pos[idx].astype(np.float32), sh[idx], rot[idx].astype(np.float32), so[idx].astype(np.float32))
    return cloud, idx


def place(rng, sizes, tiles=TILES):
    """Unclipped rectangles of the given (w, h) sizes at random positions on the grid."""
    sz = np.asarray(sizes, np.int64).reshape(-1, 2)
    tx0 = (rng.random(len(sz)) * (tiles - sz[:, 0] + 1)).astype(np.int64)
    ty0 = (rng.random(len(sz)) * (tiles - sz[:, 1] + 1)).astype(np.int64)
    return np.stack([tx0, ty0, sz[:, 0], sz[:, 1], np.zeros(len(sz), np.int64)], 1)


def clipped_rects(rng, tiles=TILES):
    """Splats clipped by each frame edge, whose clamped footprint is 4, 5, 128 or 129 tiles."""
    out = []
    for side in (LEFT, RIGHT, TOP, BOTTOM):
        for w, h in ((2, 2), (1, 5), (8, 16), (3, 43)) if side in (LEFT, RIGHT) else ((2, 2), (5, 1), (16, 8), (43, 3)):
            tx0 = 0 if side == LEFT else (tiles - w if side == RIGHT else int(rng.integers(0, tiles - w + 1)))
            ty0 = 0 if side == TOP else (tiles - h if side == BOTTOM else int(rng.integers(0, tiles - h + 1)))
            out.append((tx0, ty0, w, h, side))
    return np.array(out, np.int64)


def tiles_of(rects):
    return rects[:, 2] * rects[:, 3]


def classes_of(tiles):
    return np.where(tiles > KP.BIN_BIG, 2, np.where(tiles > KP.BIN_TINY, 1, 0))     # 0 tiny, 1 medium, 2 large


def round_boundaries(n_vis):
    return [(n_vis * f) >> 16 for f in ROUND_FRACS]


def with_boundary_runs(rects, rng):
    """Medium and large splats alternate over the ranks [b - 2, b + 2) around each inner round boundary b."""
    rects = rects.copy()
    for b in round_boundaries(len(rects)):
        for k, r in enumerate(range(b - 2, b + 2)):
            sizes = MEDIUM_SIZES if k % 2 == 0 else LARGE_SIZES
            rects[r] = place(rng, [sizes[int(rng.integers(len(sizes)))]])[0]
    return rects


# the cases --------------------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def case_a():
    """Class boundaries: 1..6, 128 and 129 tiles in several shapes plus the edge-clipped ones, in shuffled rank order
    among tiny filler splats (n_visible 12 000, so every inner round boundary lands on a run of medium/large ones)."""
    rng = np.random.default_rng(101)
    sizes = [(1, 1), (1, 2), (2, 1), (1, 3), (3, 1), (1, 4), (4, 1), (2, 2), (1, 5), (5, 1), (2, 3), (3, 2), (1, 6),
             (1, 128), (128, 1), (8, 16), (2, 64), (1, 129), (129, 1), (3, 43)]
    special = np.concatenate([place(rng, sizes * 8), clipped_rects(rng)])
    n = 12_000
    rects = place(rng, [TINY_SIZES[i % len(TINY_SIZES)] for i in range(n)])
    ranks = rng.choice(np.arange(40, n - 40), len(special), replace=False)
    rects[ranks] = special[rng.permutation(len(special))]
    rects = with_boundary_runs(rects, rng)
    return (*footprint_cloud(rects, seed=1), rects)


B_PARTS = (16, 8, 4, 2, 1)


def b_counts(queued):
    """(parts, n_large) at both ends of each part count's interval; for one part, the low end and a count with more
    large splats than the grid has warps."""
    grid = KP.bin_grid(SM, queued)
    warps = grid * KP.BIN_WARPS_PER_CTA
    out = []
    for p in B_PARTS:
        inside = [nl for nl in range(1, warps + 1) if KP.large_split_parts(nl, grid) == p]
        out += [(p, inside[0]), (p, inside[-1] if p > 1 else warps + 37)]
    return out


B_CASES = [(q, p, nl) for q in (False, True) for p, nl in b_counts(q)]


@functools.lru_cache(maxsize=None)
def case_b(n_large):
    rng = np.random.default_rng(200 + n_large)
    rects = place(rng, [LARGE_SIZES[i % len(LARGE_SIZES)] for i in range(n_large)])
    return (*footprint_cloud(rects, seed=n_large), rects)


C_CASES = [(q, n) for q in (False, True) for n in (20, 1000, 32 * KP.bin_grid(SM, q) * KP.BIN_WARPS_PER_CTA + 1000)]


@functools.lru_cache(maxsize=None)
def case_c(n_med):
    rng = np.random.default_rng(300 + n_med)
    rects = place(rng, [MEDIUM_SIZES[i % len(MEDIUM_SIZES)] for i in range(n_med)])
    return (*footprint_cloud(rects, seed=n_med), rects)


D_N = 300_000


@functools.lru_cache(maxsize=None)
def case_d():
    """300 000 splats: a large one every 50 ranks and a medium one every 10, offset so that every 2048-rank sub-tile of
    every queued CTA holds all three classes; runs of medium/large splats on the round boundaries."""
    rng = np.random.default_rng(400)
    r = np.arange(D_N)
    cls = np.where(r % 50 == 7, 2, np.where(r % 10 == 3, 1, 0))
    sizes = np.empty((D_N, 2), np.int64)
    for c, pal in enumerate((TINY_SIZES, MEDIUM_SIZES, LARGE_SIZES)):
        m = cls == c
        sizes[m] = np.asarray(pal)[rng.integers(0, len(pal), int(m.sum()))]
    rects = with_boundary_runs(place(rng, sizes), rng)
    return (*footprint_cloud(rects, seed=4, d0=2.5, d1=30.0), rects)


CAP0 = KP.initial_pair_capacity(0)            # 2^20: the first frame's pair capacity for clouds below 2^20
F_STRADDLE = {"tiny": ((2, 2), 2), "medium": ((4, 4), 7), "large": ((43, 3), 50), "exact": ((3, 3), 0)}
F_FILL = (TILES, 8)


@functools.lru_cache(maxsize=None)
def case_f(kind):
    """Fillers (1040-tile rows and single tiles, shuffled) up to 2^20 - k pairs, then the splat of `kind` whose pairs
    start there (k pairs before the capacity; 0: it starts exactly on it), then 64 single-tile splats."""
    (w, h), k = F_STRADDLE[kind]
    rng = np.random.default_rng(500 + k)
    q, r = divmod(CAP0 - k, F_FILL[0] * F_FILL[1])
    fill = np.concatenate([place(rng, [F_FILL] * q), place(rng, [(1, 1)] * r)])
    rects = np.concatenate([fill[rng.permutation(len(fill))], place(rng, [(w, h)]), place(rng, [(1, 1)] * 64)])
    return (*footprint_cloud(rects, seed=k), rects)


G_VIEW = B.headless_view(4112, 4112)          # 66 049 tiles
G_COUNTS = {"ge_2^30": 16_300, "gt_2^32": 65_100}


def case_g(count):
    return footprint_cloud(np.tile([[0, 0, 257, 257, COVER]], (count, 1)), seed=count, view=G_VIEW, d0=3.0, d1=6.0)


def decoy_cloud(rects, seed):
    """A different, larger cloud on the same grid: the same footprints placed elsewhere, in another rank order, plus
    a quarter more medium ones; so it has more splats and more pairs than the case."""
    rng = np.random.default_rng(seed + 7)
    extra = place(rng, [MEDIUM_SIZES[i % len(MEDIUM_SIZES)] for i in range(len(rects) // 4 + 64)])
    moved = place(rng, rects[:, 2:4])
    both = np.concatenate([moved, extra])
    return footprint_cloud(both[rng.permutation(len(both))], seed=seed + 11)[0]


# oracle checks of the constructions (no GPU) -------------------------------------------------------------------------

def oracle_footprints(oracle, cloud, view=VIEW):
    """-> (rank_to_id, (n_vis, 4) tile rectangles by rank) from the oracle's keys and projection."""
    keys = oracle.keygen(cloud.position_visibility, view.to_abi(), UNIFORM, 32)
    _, order = oracle.radix_sort(keys, 32)
    n_vis = int((keys != 0xFFFFFFFF).sum())
    r2i = np.ascontiguousarray(order[:n_vis][::-1])          # ascending keys run far to near; rank 0 is the nearest
    rec = oracle.project(cloud, view.to_abi(), UNIFORM, S.to_abi(), r2i)
    bx = np.stack([rec["xlo"], rec["xhi"], rec["ylo"], rec["yhi"]], 1)
    return r2i, np.array([KP.footprint_rect(*map(int, b)) for b in bx], np.int64).reshape(-1, 4)


def check_construction(oracle, cloud, idx, rects, view=VIEW):
    r2i, got = oracle_footprints(oracle, cloud, view)
    assert len(r2i) == len(rects), "every splat must be visible"
    assert np.array_equal(r2i, np.argsort(idx)), "the rank order must be the planned one"
    bad = np.flatnonzero(np.any(got != rects[:, :4], 1))
    assert len(bad) == 0, f"{len(bad)} footprints off, e.g. rank {bad[:3]}: {got[bad[:3]]} != {rects[bad[:3], :4]}"
    return got


def test_class_boundary_construction(oracle):
    cloud, idx, rects = case_a()
    got = check_construction(oracle, cloud, idx, rects)
    t = tiles_of(got)
    for v in (1, 2, 3, 4, 5, 6, 128, 129):
        assert np.any(t == v), v
    shapes = {tuple(x) for x in got[:, 2:4]}
    assert {(1, 4), (4, 1), (2, 2), (1, 5), (5, 1), (1, 128), (128, 1), (8, 16), (2, 64), (1, 129), (129, 1), (3, 43)} <= shapes
    # edge-clipped splats, clamped to 4, 5, 128 and 129 tiles at every edge
    clipped = rects[:, 4] != NONE
    assert {(int(c), int(v)) for c, v in zip(rects[clipped, 4], t[clipped])} == \
        {(c, v) for c in (LEFT, RIGHT, TOP, BOTTOM) for v in (4, 5, 128, 129)}
    lo = (got[:, 0] == 0) | (got[:, 1] == 0)
    hi = (got[:, 0] + got[:, 2] == TILES) | (got[:, 1] + got[:, 3] == TILES)
    assert np.all((lo | hi)[clipped])
    cls = classes_of(t)
    assert all(np.any(cls == c) for c in range(3))
    for b in round_boundaries(len(rects)):
        assert b >= 2 and set(cls[b - 2:b + 2]) == {1, 2}, b


@pytest.mark.parametrize("queued,parts,n_large", B_CASES)
def test_large_split_construction(oracle, queued, parts, n_large):
    grid = KP.bin_grid(SM, queued)
    assert KP.large_split_parts(n_large, grid) == parts
    cloud, idx, rects = case_b(n_large)
    got = check_construction(oracle, cloud, idx, rects)
    assert np.all(classes_of(tiles_of(got)) == 2)
    if n_large > grid * KP.BIN_WARPS_PER_CTA:
        assert KP.large_tickets(n_large, grid)[1] == 2


def test_large_split_constructions_reach_every_slice_shape():
    """Across the split cases: empty trailing parts, a one-pair last part, a footprint that is a multiple of `per`,
    one of per * parts - 1 pairs, parts that start mid-row, and every width phase 3b's row step must handle."""
    seen = set()
    widths = set()
    for queued, parts, n_large in B_CASES:
        rects = case_b(n_large)[2]
        for w, h in {tuple(x) for x in rects[:, 2:4]}:
            widths.add(int(w))
            total = int(w * h)
            sl = KP.large_part_slices(total, parts)
            per = sl[0][1] - sl[0][0] if parts > 1 else total
            if any(a >= total for a, _ in sl):
                seen.add(("empty", parts))
            if any(b - a == 1 for a, b in sl):
                seen.add(("one pair", parts))
            if parts > 1 and total % per == 0 and total == per * parts:
                seen.add(("multiple of per", parts))
            if parts > 1 and total == per * parts - 1:
                seen.add(("per*parts-1", parts))
            if any(a < total and a % w for a, _ in sl):
                seen.add(("mid-row", parts))
    for p in (16, 8, 4, 2):
        assert {("multiple of per", p), ("per*parts-1", p), ("mid-row", p)} <= seen, p
    assert ("empty", 16) in seen and ("one pair", 16) in seen
    assert KP.large_part_slices(129, 16)[4] == (128, 129) and KP.large_part_slices(513, 16)[8] == (512, 513)
    assert {1, 2, 31, 32, 33, 64, 65, TILES} <= widths


@pytest.mark.parametrize("queued,n_med", C_CASES)
def test_medium_drain_construction(oracle, queued, n_med):
    grid = KP.bin_grid(SM, queued)
    cloud, idx, rects = case_c(n_med)
    got = check_construction(oracle, cloud, idx, rects)
    assert np.all(classes_of(tiles_of(got)) == 1)
    assert KP.medium_passes(n_med, grid) == (2 if n_med > 1000 else 1)
    assert n_med < 32 or n_med % 32


def cta_subtile_classes(cls, grid):
    """For each binning CTA, the set of footprint classes in each of its sub-tiles."""
    return [[set(cls[a:b].tolist()) for a, b in subs] for subs in KP.bin_subtiles(len(cls), grid)]


def test_mixed_subtile_construction(oracle):
    cloud, idx, rects = case_d()
    got = check_construction(oracle, cloud, idx, rects)
    cls = classes_of(tiles_of(got))
    grid = KP.bin_grid(SM, queued=True)
    assert KP.bin_multi_subtile(D_N, grid) and D_N > 270_000
    for subs in cta_subtile_classes(cls, grid):
        assert sum(s == {0, 1, 2} for s in subs) >= 2
    for b in round_boundaries(D_N):
        assert set(cls[b - 2:b + 2]) == {1, 2}, b


@pytest.mark.parametrize("kind", list(F_STRADDLE))
def test_capacity_crossing_construction(oracle, kind):
    cloud, idx, rects = case_f(kind)
    got = check_construction(oracle, cloud, idx, rects)
    t = tiles_of(got)
    off = np.concatenate([[0], np.cumsum(t)])
    (w, h), k = F_STRADDLE[kind]
    r = len(rects) - 65                                    # the straddling splat's rank
    assert len(cloud) < CAP0 and KP.initial_pair_capacity(len(cloud)) == CAP0 and off[-1] > CAP0
    assert off[r] == CAP0 - k and t[r] == w * h
    if kind == "exact":
        assert off[r] == CAP0
    else:
        assert off[r] < CAP0 < off[r + 1] and KP.footprint_class(int(t[r])) == kind


@pytest.mark.parametrize("name", list(G_COUNTS))
def test_pair_limit_construction(oracle, name):
    count = G_COUNTS[name]
    cloud, _ = case_g(count)
    tiles = KP.num_tiles(G_VIEW.width, G_VIEW.height)
    rec = oracle.project(cloud, G_VIEW.to_abi(), UNIFORM, S.to_abi(), np.arange(count, dtype=np.uint32))
    keys = oracle.keygen(cloud.position_visibility, G_VIEW.to_abi(), UNIFORM, 32)
    assert np.all(keys != 0xFFFFFFFF)
    assert np.all(rec["xlo"] == 0) and np.all(rec["ylo"] == 0)
    assert np.all(rec["xhi"] == G_VIEW.width - 1) and np.all(rec["yhi"] == G_VIEW.height - 1)
    need = count * tiles
    assert tiles == 66_049 and need >= (1 << 30) - 1
    if name == "gt_2^32":
        assert need > 1 << 32


# ---------------------------------------------------------------------------------------------------------------------
# GPU cases

def assert_tiles_match(p, til):
    fs = p.frame_stats()
    assert fs.rounds == 1
    assert fs.n_visible == til["n_vis"] and fs.n_pairs == til["n_pairs"], (fs.n_visible, fs.n_pairs, til["n_vis"], til["n_pairs"])
    _, ids = p.projected()
    assert np.array_equal(ids, til["rank_to_id"]), "rank order differs"
    assert np.array_equal(p.tile_ranges(), til["tile_ranges"]), "tile ranges differ (must be bit-exact)"
    got = p.tile_entries()
    bad = np.flatnonzero(got != til["tile_entries"])
    assert len(bad) == 0, f"{len(bad)} tile entries differ, first at {bad[:4]}"


def run_case(oracle, cloud, rects, queued, decoy_seed, image=False, rounds_too=False):
    """Decoy frame, then the case in the same context; -> the case's frame (host rgba32f when `image`)."""
    assert KP.device_sm_count() == SM, "the cases are sized for 132 SMs"
    p = B.GaussianSplattingPlugin(0)
    try:
        decoy = decoy_cloud(rects, decoy_seed)
        assert len(decoy) > len(cloud) and KP.num_tiles(VIEW.width, VIEW.height) == TILES * TILES
        hd = p.add_cloud(decoy)
        render_frame(p, hd, S, VIEW, queued)
        decoy_pairs = p.frame_stats().n_pairs
        hd.destroy()
        h = p.add_cloud(cloud)
        try:
            til = oracle.render_tiles(cloud, VIEW.to_abi(), p.cloud_uniform(S, None, h.aabb), S.to_abi(), want_image=image)
            assert decoy_pairs >= til["n_pairs"], "the decoy must fill every pair slot of the case"
            img = render_frame(p, h, S, VIEW, queued)
            assert_tiles_match(p, til)
            if image:
                err = float(np.abs(img - til["image"]).max())
                assert err <= PIXEL_TOL, f"pixel L-inf {err}"
            if rounds_too:
                fs1 = p.frame_stats()
                many = render_frame(p, h, S_ROUNDS, VIEW, queued)
                fs2 = p.frame_stats()
                assert fs2.rounds == 5 and fs2.n_visible == fs1.n_visible
                if fs2.tiles_saturated < fs2.tiles_x * fs2.tiles_y:
                    assert fs2.n_pairs == fs1.n_pairs        # every round emitted
                assert np.array_equal(many.view(np.uint8), img.view(np.uint8)), "binning rounds changed the frame"
            return img, til
        finally:
            h.destroy()
    finally:
        p.destroy()


@gpu
@pytest.mark.parametrize("queued", MODES)
def test_class_boundaries_vs_oracle(oracle, queued):
    """(a) Footprints of 1..6, 128 and 129 tiles in several shapes and clipped by each frame edge, overlapping and
    shuffled in rank order: pixels within the bar too."""
    cloud, _, rects = case_a()
    cls = classes_of(tiles_of(rects))
    assert all(np.any(cls == c) for c in range(3))
    run_case(oracle, cloud, rects, queued, 1, image=True)


@gpu
@pytest.mark.parametrize("queued,parts,n_large", B_CASES)
def test_large_footprint_splits_vs_oracle(oracle, queued, parts, n_large):
    """(b) Every part count at both ends of its interval for the grid in use, and more large splats than warps."""
    grid = KP.bin_grid(KP.device_sm_count(), queued)
    p_got, per_warp = KP.large_tickets(n_large, grid)
    assert p_got == parts and per_warp == (2 if n_large > grid * KP.BIN_WARPS_PER_CTA else 1)
    cloud, _, rects = case_b(n_large)
    run_case(oracle, cloud, rects, queued, 2 + n_large)


@gpu
@pytest.mark.parametrize("queued,n_med", C_CASES)
def test_medium_drain_passes_vs_oracle(oracle, queued, n_med):
    """(c) Fewer than 32 medium splats, a count that is not a multiple of 32, and more than one pass per warp."""
    grid = KP.bin_grid(KP.device_sm_count(), queued)
    assert KP.medium_passes(n_med, grid) == (2 if n_med > 1000 else 1)
    cloud, _, rects = case_c(n_med)
    run_case(oracle, cloud, rects, queued, 3 + n_med)


@gpu
@pytest.mark.parametrize("queued", MODES)
def test_mixed_classes_across_subtiles_vs_oracle(oracle, queued):
    """(d) 300 000 splats of all three classes: a queued frame's 132 CTAs each bin two sub-tiles that both hold every
    class, so the medium and large queue positions are carried from one sub-tile to the next."""
    grid = KP.bin_grid(KP.device_sm_count(), queued)
    cloud, _, rects = case_d()
    if queued:
        assert KP.bin_multi_subtile(D_N, grid)
        for subs in cta_subtile_classes(classes_of(tiles_of(rects)), grid):
            assert sum(s == {0, 1, 2} for s in subs) >= 2
    run_case(oracle, cloud, rects, queued, 4)


@gpu
@pytest.mark.parametrize("queued", MODES)
@pytest.mark.parametrize("which", ["a", "d"])
def test_binning_rounds_split_class_runs(oracle, which, queued):
    """(e) Binning rounds whose boundaries fall inside runs of medium and large splats: byte-identical to the one-round
    frame, which matches the oracle."""
    cloud, _, rects = case_a() if which == "a" else case_d()
    cls = classes_of(tiles_of(rects))
    for b in round_boundaries(len(rects)):
        assert set(cls[b - 2:b + 2]) == {1, 2}
    assert KP.chunked(TILES * TILES, flag=True)
    run_case(oracle, cloud, rects, queued, 5, rounds_too=True)


@gpu
@pytest.mark.parametrize("queued", MODES)
@pytest.mark.parametrize("kind", list(F_STRADDLE))
def test_capacity_crossing_vs_oracle(oracle, kind, queued):
    """(f) The first frame of a fresh context needs more than its 2^20-pair buffer, and the capacity falls inside a
    tiny, a medium or a large footprint's pairs, or exactly on a footprint's start.  The truncated pass itself cannot
    be observed (its pairs are overwritten when the frame is redone in the grown buffer): what is checked is that the
    overflow is detected and that the redone frame matches the oracle.  No decoy: the frame must be the context's
    first."""
    cloud, _, rects = case_f(kind)
    p = B.GaussianSplattingPlugin(0)
    try:
        h = p.add_cloud(cloud)
        til = oracle.render_tiles(cloud, VIEW.to_abi(), p.cloud_uniform(S, None, h.aabb), S.to_abi(), want_image=False)
        assert til["n_pairs"] > KP.initial_pair_capacity(len(cloud))
        if queued:
            p.render_view(h, S, VIEW, to_host=False, asynchronous=True)
            assert not p.sync(), "the first frame must outgrow the pair buffer"
            p.render_view(h, S, VIEW, to_host=False, asynchronous=True)
            assert p.sync()
        else:
            p.render_view(h, S, VIEW, to_host=False)
        assert_tiles_match(p, til)
        h.destroy()
    finally:
        p.destroy()


@gpu
@pytest.mark.parametrize("queued", MODES)
@pytest.mark.parametrize("name", list(G_COUNTS))
def test_pair_count_limit_refused(oracle, name, queued):
    """(g) Splats that each cover all 66 049 tiles of a 4112 x 4112 frame: 16 300 of them need more than 2^30 - 1
    pairs, 65 100 more than 2^32 (the count must saturate, not wrap).  Both frames are refused with BGS_ENOMEM, a host
    status (nothing near 2^30 pairs is allocated), and the context then renders a normal frame."""
    cloud, _ = case_g(G_COUNTS[name])
    p = B.GaussianSplattingPlugin(0)
    try:
        h = p.add_cloud(cloud)
        with pytest.raises(abi.BgsError, match=r"2\^30") as e:
            if queued:
                p.render_view(h, S, G_VIEW, to_host=False, asynchronous=True)
                p.sync()
            else:
                p.render_view(h, S, G_VIEW, to_host=False)
        assert e.value.status == abi.BGS_ENOMEM
        h.destroy()
        check_against_oracle(p, oracle, B.random_gaussians_3d_seeded(20_000, 3), B.CloudSettings(global_scale=0.25),
                             B.headless_view(320, 200), asynchronous=queued)
    finally:
        p.destroy()
