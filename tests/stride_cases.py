"""Inputs of the striding tests (tests/test_gpu_strides.py, tests/test_oracle_strides.py): frames whose projection and
splat-depth loops take many grid-stride passes, and scenes whose key-gen carries segments across warps, tiles, chunks
and CTA ranges.

A context plans its projection grid from the previous completed frame's visible count (kernel_paths.projection_hint).
After a frame with exactly one visible gaussian (`starve_cloud`) the next frame's hint is 1025: a 9-CTA projection grid
and a 5-CTA splat-depth grid, whatever that frame's size.  A frame of a few thousand to tens of thousands of visible
splats then takes several to dozens of passes per warp, with a cloud small enough for the CPU oracles.

* A `single_cloud`: one 3D cloud at SH degree 0..3, about 31 500 of 36 000 gaussians visible.
* B `performer_4d`: one Gaussian4d cloud, about 40 % of its visible splats masked by time at STRIDE_4D_TIMES.
* C `mixed_clouds` / `mixed_segments`: eight 3D clouds (f32 and f16 at degree 0..3) and a 4D one, cut into 64 segments and interleaved.
* D `keygen_scene_layout`: 64 segments over N = 4 700 001 gaussians, boundaries placed on and around every unit the
  scene key-gen walks (32 items, 2048-gaussian tiles, 32 768-gaussian phase-2 chunks, CTA ranges).
"""
from __future__ import annotations

import numpy as np

import bevy_gaussian_splatting_b200 as B
import kernel_paths as KP
import scene4d_cases as S4
import scene_cases as SC

f32 = np.float32
RM = B.RasterizeMode

STRIDE_VIEW = B.headless_view(256, 192)
PREV_VIEW = B.perspective_view((0.05, 1.45, 5.1), (0.0, 1.5, 4.0), 256, 192)   # OpticalFlow's previous camera
NUM_CLASSES = 5
SINGLE_N = 36_000
STARVED_HINT = KP.projection_hint(1, 1 << 30)     # 1025


def starve_cloud() -> B.PlanarGaussian3d:
    """One small gaussian on the view axis: a frame of it has exactly one visible splat on one tile, so the context's
    next frame plans for projection_hint(1, n) = 1025 records (and for one visible splat and one tile's pairs in every
    other stage)."""
    return B.PlanarGaussian3d(np.array([[0.0, 1.5, 0.0, 1.0]], f32), np.zeros((1, 48), f32),
                              np.array([[1.0, 0.0, 0.0, 0.0]], f32), np.array([[0.01, 0.01, 0.01, 0.5]], f32))


def _behind(pos: np.ndarray, every: int, phase: int = 0) -> np.ndarray:
    """Moves every `every`-th gaussian behind the camera (z > 5): culled by key-gen, interleaved with visible ones."""
    pos = pos.copy()
    pos[phase::every, 2] = np.abs(pos[phase::every, 2]) + f32(6.0)
    return pos


def single_cloud(d: int, seed: int = 0, n: int = SINGLE_N) -> B.PlanarGaussian3d:
    """n gaussians at SH degree d in front of the camera, every 8th culled; visibility lanes hold labels 0..4 (drawn by
    DrawMode::All, coloured by Classification)."""
    c = SC.cloud_in_box(n, 500 + seed, centre=(0.0, 1.5, -1.0), half=1.4, scale=0.05, sh_degree=d)
    pos = _behind(c.position_visibility, 8, 3)
    pos[:, 3] = np.random.default_rng(seed).integers(0, NUM_CLASSES, n).astype(f32)
    return B.PlanarGaussian3d(pos, c.spherical_harmonic, c.rotation, c.scale_opacity)


def single_modes(layout: str) -> list[tuple[str, RM | None]]:
    """(name, mode) of every single-cloud frame a layout takes; mode None is bgs_render_aux (colour, depth, normal).
    The covariance layout has no rotation: no Normal, no aux."""
    modes = [("color", RM.Color), ("depth", RM.Depth), ("normal", RM.Normal), ("position", RM.Position),
             ("classification", RM.Classification), ("flow", RM.OpticalFlow), ("aux", None)]
    return [m for m in modes if layout != "cov" or m[0] not in ("normal", "aux")]


STRIDE_4D_TIMES = (0.35, 0.7)


def performer_4d(seed: int = 0, n: int = SINGLE_N) -> B.PlanarGaussian4d:
    """A Gaussian4d cloud in front of the camera, every 8th culled, labels 0..4 in the visibility lanes; timescales of
    0.04 to 0.2 over timestamps in [0, 1), so that about 40 % of the visible splats are masked at STRIDE_4D_TIMES."""
    c = S4.performer(n, 600 + seed, centre=(0.0, 1.5, -1.0), spread=1.4, scale=0.05)
    pos = _behind(c.position_visibility, 8, 5)
    pos[:, 3] = np.random.default_rng(seed).integers(0, NUM_CLASSES, n).astype(f32)
    _, sh, rot8, so, tt = c.planes()
    tt = tt.copy()
    tt[:, 1] *= f32(0.2)
    return B.PlanarGaussian4d(pos, sh, rot8, so, tt)


MODES_4D = [RM.Color, RM.Depth, RM.Position, RM.Classification, RM.OpticalFlow, RM.Velocity]


# ---------------------------------------------------------------------------------------------------------------------
# C: one scene of every projection group

MIXED_LAYOUTS = [("f32", 0), ("f16", 0), ("f32", 1), ("f16", 1), ("f32", 2), ("f16", 2), ("f32", 3), ("f16", 3), ("4d", 3)]
MIXED_PIECES = 7      # segments per cloud (cloud 0 has one more: 64 in all)
MIXED_N = 600
MIXED_WINDOW = (-0.2, 1.1)
MIXED_TIME = 0.45


def mixed_group(layout: str, d: int) -> int:
    """project.cu:768-771 (project_group): the projection launch a cloud's segments belong to."""
    return KP_GROUP_4D if layout == "4d" else (1 if layout == "f16" else 0) | d << 1


KP_GROUP_4D = 8       # common.cuh:71 PROJECT_GROUP_4D


def mixed_clouds(seed: int = 0):
    """[(layout, degree, host cloud, transform, settings overrides)] of the nine clouds: each its own transform and
    global_scale."""
    out = []
    for j, (layout, d) in enumerate(MIXED_LAYOUTS):
        if layout == "4d":
            c = S4.performer(MIXED_N, 700 + seed, centre=(0.0, 1.5, -1.0), spread=1.3, scale=0.07)
            pos = _behind(c.position_visibility, 9, 4)
            c = B.PlanarGaussian4d(pos, *c.planes()[1:])
        else:
            c = SC.cloud_in_box(MIXED_N, 710 + 10 * seed + j, centre=(0.0, 1.5, -1.0), half=1.3, scale=0.07, sh_degree=d)
            pos = _behind(c.position_visibility, 9, j % 9)
            pos[:, 3] = np.random.default_rng(j).integers(0, NUM_CLASSES, MIXED_N).astype(f32)
            c = B.PlanarGaussian3d(pos, c.spherical_harmonic, c.rotation, c.scale_opacity)
        tr = SC.transform((0.04 * (j - 4), 0.03 * (j % 3 - 1), -0.05 * (j % 2)), 0.9 + 0.03 * j, 0.1 * (j - 4))
        kw = dict(global_scale=0.8 + 0.06 * j, global_opacity=1.0 - 0.03 * j)
        out.append((layout, d, c, tr, kw))
    return out


def mixed_segments(seed: int = 0) -> list[tuple[int, np.ndarray]]:
    """64 segments (cloud j, its contiguous index range), interleaved round-robin over the nine clouds."""
    per = [SC.pieces(MIXED_N, MIXED_PIECES + (1 if j == 0 else 0), 50 + j + seed) for j in range(len(MIXED_LAYOUTS))]
    segs = []
    for i in range(MIXED_PIECES + 1):
        for j, ps in enumerate(per):
            if i < len(ps):
                segs.append((j, ps[i]))
    assert len(segs) == 64
    return segs


# ---------------------------------------------------------------------------------------------------------------------
# D: key-gen at scale

KEYGEN_N = 4_700_001                      # > 132 x 17 x 2048: every queued key-gen CTA owns at least 17 tiles
KEYGEN_PERIOD = 60 * 10_007               # positions repeat with this period: equal keys in many segments
KEYGEN_WARP_RUN = (1, 2, 5, 31)           # segments inside one warp's items


def keygen_positions(n: int = KEYGEN_N, seed: int = 7) -> np.ndarray:
    """(n, 4) positions, 1 in 60 in the frustum of STRIDE_VIEW (2 to 20 units away), the rest behind
    the camera, periodic in KEYGEN_PERIOD; around each segment of the warp run some culled ones are made visible."""
    rng = np.random.default_rng(seed)
    per = np.empty((KEYGEN_PERIOD, 4), f32)
    per[:, :3] = rng.uniform(-20, 20, (KEYGEN_PERIOD, 3)).astype(f32)
    per[:, 2] = np.abs(per[:, 2]) + f32(5.5)
    per[:, 3] = 1.0
    vis = np.arange(0, KEYGEN_PERIOD, 60)
    dist = rng.uniform(2.0, 20.0, len(vis)).astype(f32)
    per[vis, 0] = rng.uniform(-0.5, 0.5, len(vis)).astype(f32) * dist
    per[vis, 1] = f32(1.5) + rng.uniform(-0.35, 0.35, len(vis)).astype(f32) * dist
    per[vis, 2] = f32(5.0) - dist
    pos = np.resize(per, (n, 4))
    w0 = warp_run_start()
    for k in (0, 1, 3, 5, 9, 12, 20, 27, 33, 38):   # visible: seg 1, seg 2 (first), seg 5 (two), seg 31 (five)
        pos[w0 + k] = per[vis[k + 1]]
    return pos


def warp_run_start() -> int:
    return 999_936                           # a multiple of 256: the first item of a warp's 8 x 32


def keygen_targets(n: int = KEYGEN_N, sm: int = KP.H100_SMS) -> dict[str, list[int]]:
    """Where segment boundaries must lie: name -> cut positions (global indices where a segment starts)."""
    tiles = KP.keygen_cta_tiles(n, sm)
    w0 = warp_run_start()
    run = [w0]
    for L in KEYGEN_WARP_RUN:
        run.append(run[-1] + L)
    item = 1_500_000                         # a multiple of 32, not of 2048
    tile = 2048 * 1200
    chunk = tiles[20][0] * KP.KG_TILE + KP.KG_CHUNK_TILES * KP.KG_TILE    # CTA 20's second phase-2 chunk
    cta = tiles[100][0] * KP.KG_TILE                                      # CTA 100's first gaussian
    return {"warp_run": run, "item": [item - 1, item, item + 1], "tile": [tile - 1, tile, tile + 1],
            "chunk": [chunk - 1, chunk, chunk + 1], "cta": [cta - 1, cta, cta + 1]}


def keygen_scene_layout(n: int = KEYGEN_N, sm: int = KP.H100_SMS, segments: int = 64) -> list[tuple[int, int]]:
    """The 64 segments [a, b) of [0, n): every target cut, and the rest of [0, n) cut evenly between them."""
    must = sorted({c for cs in keygen_targets(n, sm).values() for c in cs})
    free = segments - (len(must) + 1)
    # spread the remaining cuts over the gaps, in proportion to their lengths
    edges = [0] + must + [n]
    gaps = [(edges[i + 1] - edges[i], i) for i in range(len(edges) - 1)]
    total = sum(g for g, _ in gaps)
    extra = {i: int(free * g / total) for g, i in gaps}
    left = free - sum(extra.values())
    for g, i in sorted(gaps, reverse=True)[:left]:
        extra[i] += 1
    cuts = []
    for i in range(len(edges) - 1):
        a, b = edges[i], edges[i + 1]
        k = extra[i]
        cuts += [a + (b - a) * (m + 1) // (k + 1) for m in range(k)]
    allc = sorted(set(must + cuts))
    bounds = [0] + allc + [n]
    segs = list(zip(bounds[:-1], bounds[1:]))
    assert len(segs) == segments and all(b > a for a, b in segs), len(segs)
    return segs


def keygen_uniform_index(j: int, a: int) -> int:
    """Which of keygen_transforms() segment j (starting at a) gets: the warp run's segments each their own, every other
    segment one of three in turn.  Segments three apart share a uniform, and the positions repeat: equal keys meet
    across segments all over the frame."""
    w0 = warp_run_start()
    if w0 <= a < w0 + sum(KEYGEN_WARP_RUN):
        return 3 + [w0 + sum(KEYGEN_WARP_RUN[:i]) for i in range(4)].index(a)
    return j % 3


def keygen_transforms():
    """Seven small rigid transforms and global scales: each keeps the visible gaussians in the frustum."""
    out = []
    for i in range(7):
        out.append((SC.transform((0.03 * (i - 3), 0.02 * (i % 2), 0.04 * (i % 3)), 1.0 + 0.01 * i, 0.01 * (i - 3)),
                    0.8 + 0.05 * i))
    return out
