"""Each case of test_gpu_strides.py reaches the path it exists for (no GPU): the selection rules of kernel_paths applied to
the visible sets the CPU oracles' key-gen finds.  If the library's rules change, these fail instead of coverage moving
silently."""
import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import kernel_paths as KP
import stride_cases as SD
import temporal_cases as TC
from scene_oracle import scene_oracle as SO

VIEW = SD.STRIDE_VIEW
CULLED = 0xFFFFFFFF
STARVED_GRID = KP.project_grid(SD.STARVED_HINT)
MIN_PASSES = 3


def visible(oracle, pos, uniform=None):
    u = uniform if uniform is not None else B.GaussianSplattingPlugin.cloud_uniform(B.CloudSettings())
    return oracle.keygen(np.ascontiguousarray(pos), VIEW.to_abi(), u, 32) != CULLED


def test_starved_frame_geometry():
    assert SD.STARVED_HINT == 1025 and KP.projection_hint(0, 36_000) == 36_000
    assert KP.projection_hint(31_000, 36_000) == 36_000 and KP.projection_hint(20_000, 36_000) == 26_024
    assert STARVED_GRID == 9 and KP.splat_depth_grid(SD.STARVED_HINT) == 5
    assert KP.project_grid(10_000_000) == 4 * KP.H100_SMS and KP.splat_depth_grid(10_000_000) == 8 * KP.H100_SMS
    assert KP.project_passes(1152, 9) == 1 and KP.project_passes(1153, 9) == 2 and KP.project_min_passes(1153, 9) == 1
    assert KP.project_min_passes(3425, 9) == 3 and KP.project_min_passes(3424, 9) == 2
    # a fresh frame's capped grid (528 CTAs, 67 584 entries a pass) strides past 67 584 visible, twice past 135 168
    assert KP.project_grid(135_169) == 528 and KP.project_passes(67_584, 528) == 1 and KP.project_passes(67_585, 528) == 2
    assert KP.project_passes(135_168, 528) == 2 and KP.project_passes(135_169, 528) == 3
    assert KP.scene_keygen_grid(True) == KP.H100_SMS
    assert all(KP.scene_keygen_grid(False, KP.H100_SMS, 4, fit) <= 4 * KP.H100_SMS for fit in range(1, 9))
    t = KP.keygen_cta_tiles(SD.KEYGEN_N, 7)
    assert t[0][0] == 0 and t[-1][1] == -(-SD.KEYGEN_N // KP.KG_TILE) and all(a[1] == b[0] for a, b in zip(t, t[1:]))


@pytest.mark.parametrize("d", [0, 1, 2, 3])
def test_single_clouds_stride(oracle, d):
    cloud = SD.single_cloud(d, d)
    vis = visible(oracle, cloud.position_visibility)
    nv, n = int(vis.sum()), len(cloud)
    assert KP.project_min_passes(nv, STARVED_GRID) >= 20
    assert KP.splat_depth_passes(nv, KP.splat_depth_grid(SD.STARVED_HINT)) >= 20
    # the fresh frame strides once: the three ways take different paths to the same frame
    assert KP.project_passes(nv, KP.project_grid(KP.projection_hint(0, n))) == 1
    assert KP.project_passes(nv, KP.project_grid(KP.projection_hint(nv, n))) == 1
    assert 0.8 * n < nv < n     # visible and culled interleaved


def test_4d_cloud_strides_with_mixed_masks(oracle):
    cloud = SD.performer_4d(0)
    vis = visible(oracle, cloud.position_visibility)
    nv = int(vis.sum())
    assert KP.project_min_passes(nv, STARVED_GRID) >= 20
    for t in SD.STRIDE_4D_TIMES:
        _, _, _, mask = TC.condition(cloud.isotropic_rotations, cloud.scale_opacity, cloud.timestamp_timescale, 1.0, t)
        masked = ~mask[vis]
        assert 0.25 <= masked.mean() <= 0.75, masked.mean()
        # drawn and undrawn lanes in every group of 32 slots
        groups = masked[: nv // 32 * 32].reshape(-1, 32)
        assert (groups.any(1) & ~groups.all(1)).all()


def _mixed_slots(oracle):
    """(slot -> cloud j, slot -> segment k, n_vis, sorted entries) of the mixed scene."""
    clouds, segs = SD.mixed_clouds(), SD.mixed_segments()
    listed, cloud_of, seg_of = [], [], []
    for k, (j, ix) in enumerate(segs):
        layout, _, c, tr, kw = clouds[j]
        st = B.CloudSettings(**kw)
        u = B.GaussianSplattingPlugin.cloud_uniform(st, tr, None)
        pos = c.position_visibility[ix]
        # key-gen reads positions only: a 4D cloud's keys are those of a 3D cloud at the same positions
        listed.append((B.PlanarGaussian3d(pos, np.zeros((len(ix), 48), np.float32), np.tile([1, 0, 0, 0], (len(ix), 1)),
                                          np.ones((len(ix), 4), np.float32)), u, False))
        cloud_of += [j] * len(ix)
        seg_of += [k] * len(ix)
    entries = SO.sorted_entries(listed, VIEW.to_abi())
    vis_ids = np.sort(entries[entries[:, 0] != CULLED, 1])
    return np.array(cloud_of)[vis_ids], np.array(seg_of), vis_ids, entries


def test_mixed_scene_interleaves_every_group(oracle):
    groups = [SD.mixed_group(layout, d) for layout, d in SD.MIXED_LAYOUTS]
    assert sorted(groups) == list(range(9))
    slot_cloud, seg_of, vis_ids, entries = _mixed_slots(oracle)
    nv = len(vis_ids)
    assert KP.project_min_passes(nv, STARVED_GRID) >= MIN_PASSES
    warps = STARVED_GRID * KP.PROJ_WARPS
    for p in range(KP.project_passes(nv, STARVED_GRID)):
        lo = p * STARVED_GRID * KP.PROJ_THREADS
        if p < MIN_PASSES:     # every group in every full pass
            assert set(slot_cloud[lo:lo + STARVED_GRID * KP.PROJ_THREADS]) == set(range(9)), p
            mixed = sum(len(set(slot_cloud[KP.project_warp_slots(nv, STARVED_GRID, w, p).start:
                                           KP.project_warp_slots(nv, STARVED_GRID, w, p).stop])) >= 2 for w in range(warps))
            assert mixed >= warps // 4, (p, mixed)   # (63 boundaries over > 3424 slots: not every warp)
    # most lanes of each launch are not its own
    assert max(np.bincount(slot_cloud, minlength=9)) < 0.2 * nv
    # Depth: the range's endpoints, sorted[1] (visible) and the last culled index, in different segments
    first = entries[1, 1]
    last = int(np.flatnonzero(entries[:, 0] == CULLED).size and entries[entries[:, 0] == CULLED, 1].max())
    assert seg_of[first] != seg_of[last]


def _keygen_keys(oracle, pos, segs):
    trs = SD.keygen_transforms()
    keys = np.empty(len(pos), np.uint32)
    for j, (a, b) in enumerate(segs):
        tr, gs = trs[SD.keygen_uniform_index(j, a)]
        u = B.GaussianSplattingPlugin.cloud_uniform(B.CloudSettings(global_scale=gs), tr, None)
        keys[a:b] = oracle.keygen(np.ascontiguousarray(pos[a:b]), VIEW.to_abi(), u, 32)
    return keys


def test_keygen_scene_layout(oracle):
    n, sm = SD.KEYGEN_N, KP.H100_SMS
    segs = SD.keygen_scene_layout(n, sm)
    assert len(segs) == 64 and segs[0][0] == 0 and segs[-1][1] == n and n % KP.KG_TILE != 0
    starts = {a for a, _ in segs}
    targets = SD.keygen_targets(n, sm)
    for name, cuts in targets.items():
        assert set(cuts) <= starts, name
    item, tile = targets["item"][1], targets["tile"][1]
    assert item % 32 == 0 and item % KP.KG_TILE and tile % KP.KG_TILE == 0
    run = targets["warp_run"]
    assert run[0] % 256 == 0 and run[3] - run[0] < 32                 # segments 1, 2 and 5 inside one item of one warp
    # queued: 132 CTAs, each with more than one phase-2 chunk; synchronous: any grid up to 528 CTAs, >= 2 tiles each
    queued_tiles = KP.keygen_cta_tiles(n, KP.scene_keygen_grid(True, sm))
    assert min(t1 - t0 for t0, t1 in queued_tiles) > KP.KG_CHUNK_TILES
    assert min(t1 - t0 for t0, t1 in KP.keygen_cta_tiles(n, 4 * sm)) >= 2
    chunk, cta = targets["chunk"][1], targets["cta"][1]
    assert any(t0 * KP.KG_TILE + KP.KG_CHUNK_TILES * KP.KG_TILE == chunk for t0, _ in queued_tiles)
    assert any(t0 * KP.KG_TILE == cta for t0, _ in queued_tiles)
    pos = SD.keygen_positions(n)
    keys = _keygen_keys(oracle, pos, segs)
    vis = keys != CULLED
    assert 60_000 < vis.sum() < 100_000
    # visible gaussians on both sides of every boundary (within two items)
    for a, _ in segs[1:]:
        assert vis[a - 64:a].any() and vis[a:a + 64].any(), a
    # the warp run mixes visible and culled inside its segments
    for lo, hi in zip(run[1:], run[2:]):
        assert vis[lo:hi].any() and not vis[lo:hi].all(), (lo, hi)
    assert vis[run[0]]
    # visible gaussians in every queued CTA's second chunk
    for t0, t1 in queued_tiles:
        a = (t0 + KP.KG_CHUNK_TILES) * KP.KG_TILE
        assert vis[a:min(t1 * KP.KG_TILE, n)].any()
    # equal keys meet across segments
    seg = np.repeat(np.arange(64), [b - a for a, b in segs])
    k, s = keys[vis], seg[vis]
    order = np.argsort(k, kind="stable")
    same = (k[order][1:] == k[order][:-1]) & (s[order][1:] != s[order][:-1])
    assert same.sum() > 1000
