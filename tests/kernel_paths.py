"""Which kernel path a frame takes, restated from libbgs's host code.

libbgs picks launch geometries and kernel variants from a frame's size, the previous frame's counts (the hints),
whether the frame is queued (BGS_FLAG_ASYNC) and how far the context's buffers have grown.  The results never depend
on that choice, so a test that renders a frame cannot tell which path it ran.  The functions below restate each rule
with the lines they mirror, so a test can assert that it reached the path it exists for: if the library's selection
changes, those assertions fail instead of coverage moving silently.

Constants are the ones in csrc/ (radix.cu, keygen.cu, bin.cu, api.cu).  Nothing here needs a GPU except
`device_sm_count`.
"""
from __future__ import annotations

from typing import NamedTuple

RS_THREADS = 512                 # radix.cu:25
RS_VARIANTS = (2, 4, 6, 8, 10, 12, 16)   # radix.cu:380-386: radix_coop_kernel<ITEMS, true>
KG_TILE = 256 * 8                # keygen.cu:18-20: gaussians per key-gen tile
KG_CHUNK_TILES = 1024 // 64      # keygen.cu:53-54: phase 2 expands 1024 mask words = 16 tiles per chunk
BIN_SUBTILE_MAX = 256 * 8        # bin.cu:12-13: BIN_THREADS * COOP_ITEMS ranks per sub-tile
BIN_TINY, BIN_BIG = 4, 128       # bin.cu:14-15: footprint classes (tiles)
BIN_WARPS_PER_CTA = 256 // 32
BIN_CTAS_PER_SM_FIT = 3          # bin.cu:266-270: bin_coop_blocks_per_sm() of the 74-register, 256-thread kernel
                                 # (registers go in 256 per warp: 80 x 256 = 20 480 per CTA, 3 fit in 65 536)
COOP_CTAS_PER_SM, COOP_CTAS_PER_SM_ASYNC = 4, 1   # api.cu: COOP_CTAS_PER_SM, COOP_CTAS_PER_SM_ASYNC
SORT_CTAS_PER_SM_ASYNC = 1       # api.cu: SORT_CTAS_PER_SM_ASYNC
RADIX_CTAS_PER_SM = 2            # radix.cu:29,336: radix_coop_blocks_per_sm() of the 82 KB / 64-register kernel
CHUNK_MAX_TILES = 65536          # api.cu: CHUNK_MAX_TILES
TILE_PX = 16                     # common.cuh:10
H100_SMS = 132


class SortPath(NamedTuple):
    items: int          # items per thread of the kernel that runs (its template ITEMS)
    match_any: bool     # radix_coop_kernel<16, false>: MATCH.ANY ranking (else the peer-mask ranking)
    grid: int           # CTAs
    waves: int          # tiles per CTA the hint plans for


def radix_status_rows(capacity: int) -> int:
    """radix.cu:313-316 (radix_num_tiles): look-back status rows for a sort of up to `capacity` entries."""
    return max(4096, capacity // (RS_THREADS * 16) + 1)


def radix_sort_path(hint: int, capacity: int, sm_count: int = H100_SMS, ctas_per_sm: int = RADIX_CTAS_PER_SM,
                    status_capacity: int | None = None) -> SortPath:
    """radix.cu:357-387 (launch_radix_sort).  `capacity`: the sort's buffer capacity; `status_capacity`: what the
    context's status rows were sized for (api.cu ensure_status: the largest cloud / pair capacity seen, default `capacity`)."""
    hint = min(hint, capacity)
    want = hint + hint // 32 + 1024

    def items_for(g):
        per_wave = g * RS_THREADS * 16
        waves = -(-want // per_wave)
        return -(-want // (g * RS_THREADS * waves)), waves

    grid = sm_count
    items, waves = items_for(grid)
    if waves > 1 and ctas_per_sm >= 2:
        grid = 2 * sm_count
        items, waves = items_for(grid)
    if waves > 3:
        items = 17
    rows = radix_status_rows(capacity if status_capacity is None else status_capacity)
    items = max(items, -(-capacity // (rows * RS_THREADS)))
    for v in RS_VARIANTS:
        if items <= v:
            return SortPath(v, False, grid, waves)
    return SortPath(16, True, grid, waves)


def depth_sort_path(n: int, n_vis_hint: int, sort_all: bool, sm_count: int = H100_SMS, status_n: int | None = None) -> SortPath:
    """api.cu plan_frame (depth_hint): the depth sort of an n-gaussian cloud.  Its hint is n for SORT_ALL frames, else
    the previous frame's visible count (n when there is none); it always runs with the synchronous CTAs per SM, queued
    or not."""
    hint = n if sort_all or n_vis_hint == 0 else n_vis_hint
    return radix_sort_path(hint, n, sm_count, RADIX_CTAS_PER_SM, status_n)


def pair_sort_path(n_pairs_hint: int, cap_pairs: int, queued: bool, sm_count: int = H100_SMS) -> SortPath:
    """api.cu plan_frame (pair_hint, pair_sort_per_sm): the tile-id sort of a one-round frame.  Its hint is the
    previous frame's pair count (the pair capacity when there is none); queued frames run SORT_CTAS_PER_SM_ASYNC CTAs
    per SM."""
    hint = n_pairs_hint if n_pairs_hint else cap_pairs
    return radix_sort_path(min(hint, cap_pairs), cap_pairs, sm_count,
                           SORT_CTAS_PER_SM_ASYNC if queued else RADIX_CTAS_PER_SM)


def initial_pair_capacity(n: int) -> int:
    """api.cu render_impl: the first frame of a context sizes the pair buffer to max(2^20, n)."""
    return max(1 << 20, n)


def grown_pair_capacity(cap_pairs: int, needed: int) -> int:
    """api.cu grow_pairs: a frame that needed more pairs than the buffer holds grows it to needed * 1.25 + 1024."""
    if needed <= cap_pairs:
        return cap_pairs
    return min(needed + needed // 4 + 1024, (1 << 30) - 1)


def pair_passes(num_tiles: int) -> int:
    """api.cu pair_passes: digit passes of the tile-id sort."""
    bits = 1
    while (1 << bits) < num_tiles:
        bits += 1
    return (bits + 7) // 8


def num_tiles(width: int, height: int) -> int:
    return -(-width // TILE_PX) * -(-height // TILE_PX)


def coop_grid(sm_count: int, ctas_per_sm_fit: int, queued: bool) -> int:
    """api.cu bgs_context_create (kg_grid, bin_grid and their _async forms): key-gen / binning grid.
    `ctas_per_sm_fit`: the kernel's occupancy (cudaOccupancy...)."""
    return sm_count * min(ctas_per_sm_fit, COOP_CTAS_PER_SM_ASYNC if queued else COOP_CTAS_PER_SM)


def keygen_multi_chunk(n: int, grid: int) -> bool:
    """keygen.cu:71,131-132: some CTA's phase 2 expands more than one 1024-word chunk (more than 16 tiles of 2048)."""
    tiles = -(-n // KG_TILE)
    return -(-tiles // grid) > KG_CHUNK_TILES


def bin_multi_subtile(n_ranks: int, grid: int) -> bool:
    """bin.cu:69-75: some CTA's rank range is longer than one sub-tile (`!single`): phase 2 reloads its bboxes."""
    return n_ranks > 0 and -(-n_ranks // grid) > BIN_SUBTILE_MAX


def bin_subtiles(n_ranks: int, grid: int) -> list[list[tuple[int, int]]]:
    """bin.cu:69-75: each CTA's rank range [rlo, rhi), cut into sub-tiles of 256 * ipt ranks."""
    ipt = min(max(-(-(-(-n_ranks // grid)) // 256), 1), 8)
    sub = 256 * ipt
    return [[(s, min(s + sub, (b + 1) * n_ranks // grid)) for s in range(b * n_ranks // grid, (b + 1) * n_ranks // grid, sub)]
            for b in range(grid)]


def footprint_class(tiles: int) -> str:
    """bin.cu:166-192: who writes a splat's pairs."""
    return "none" if tiles == 0 else ("tiny" if tiles <= BIN_TINY else ("medium" if tiles <= BIN_BIG else "large"))


def large_split_parts(n_large: int, grid: int) -> int:
    """bin.cu:235-237: into how many parts each large footprint is cut (1..16)."""
    total_warps = grid * BIN_WARPS_PER_CTA
    shift = 0
    while shift < 4 and (n_large << (shift + 2)) <= total_warps:
        shift += 1
    return 1 << shift


def bin_grid(sm_count: int, queued: bool) -> int:
    """api.cu bgs_context_create (bin_grid, bin_grid_async): binning CTAs.  Queued frames run one per SM; synchronous
    ones min(occupancy, 4) per SM."""
    return coop_grid(sm_count, BIN_CTAS_PER_SM_FIT, queued)


def medium_passes(n_med: int, grid: int) -> int:
    """bin.cu:203-205: 32-splat batches of the medium queue the busiest warp (global warp 0) drains in phase 3a."""
    batches = -(-n_med // 32)
    return -(-batches // (grid * BIN_WARPS_PER_CTA))


def large_tickets(n_large: int, grid: int) -> tuple[int, int]:
    """bin.cu:234-239: (parts per large footprint, most tickets one warp takes); tickets are dealt round-robin over
    every warp of the grid, so a warp takes a second one once there are more tickets than warps."""
    parts = large_split_parts(n_large, grid)
    return parts, -(-(n_large * parts) // (grid * BIN_WARPS_PER_CTA))


def large_part_slices(total_all: int, parts: int) -> list[tuple[int, int]]:
    """bin.cu:248-251: the pair slice [i0, end) of each part of a footprint of `total_all` tiles: `per` is the
    per-part share rounded up to 32 pairs, so the trailing parts can be short or empty (end == i0)."""
    per = ((-(-total_all // parts)) + 31) & ~31
    return [(p * per, min(total_all, p * per + per)) if p * per < total_all else (p * per, p * per) for p in range(parts)]


def footprint_rect(xlo: int, xhi: int, ylo: int, yhi: int) -> tuple[int, int, int, int]:
    """bin.cu:92-93, 180-181: the (tx0, ty0, w, h) tile rectangle of a pixel bbox; (0, 0, 0, 0) when it is empty."""
    if xlo > xhi or ylo > yhi:
        return (0, 0, 0, 0)
    tx0, ty0 = xlo // TILE_PX, ylo // TILE_PX
    return (tx0, ty0, xhi // TILE_PX - tx0 + 1, yhi // TILE_PX - ty0 + 1)


def large_footprint_raster(n_vis_hint: int, n_pairs_hint: int) -> bool:
    """api.cu plan_frame (large_fp): raster2_kernel<false> instead of MODE 0's raster_kernel (USE_OBB frames only)."""
    return n_vis_hint > 0 and n_pairs_hint >= 8 * n_vis_hint


def chunked(tiles: int, raster_mode: int = 0, aux: bool = False, flag: bool | None = None, n_vis_hint: int = 0,
            n_pairs_hint: int = 0, last_rounds: int = 1) -> bool:
    """api.cu plan_frame (rounds): binning rounds.  `flag`: True = BGS_FLAG_CHUNKS, False = BGS_FLAG_NO_CHUNKS, None = neither.
    Only USE_OBB colour frames of at most 65536 tiles are ever chunked, whatever the flag says."""
    if raster_mode != 0 or aux or tiles > CHUNK_MAX_TILES or flag is False:
        return False
    if flag:
        return True
    return (n_vis_hint > 0 and n_pairs_hint >= ((3 << 22) if last_rounds > 1 else (1 << 24))
            and n_pairs_hint >= (24 if last_rounds > 1 else 32) * n_vis_hint)


def raster_lead(start: int) -> int:
    """raster.cu PairStream::entry: leading words a tile's first bulk copy skips (its slice start rounded down to 16 B)."""
    return start & 3


PROJ_THREADS, PROJ_MIN_CTAS = 128, 4   # project.cu:665: projection CTA size and the launch bound's CTAs per SM
PROJ_WARPS = PROJ_THREADS // 32
SD_THREADS, SD_CTAS_PER_SM = 256, 8    # scene_depth.cu:13: splat-depth CTA size and its cap per SM


def projection_hint(prev_n_vis: int, n: int) -> int:
    """api.cu:175 (plan_frame n_hint): records the projection grid plans for.  The previous completed frame's visible
    count plus a quarter and 1024, at most n; n on a context's first frame (no visible count yet)."""
    return min(prev_n_vis + prev_n_vis // 4 + 1024, n) if prev_n_vis else n


def project_grid(n_hint: int, sm_count: int = H100_SMS) -> int:
    """project.cu:968, 1022, 1039, 1053 (launch_project_4d, launch_project_scene, launch_project_4d_scene,
    launch_project) through entry_src.cuh:114-119 (persistent_grid): ceil(n_hint / 128) CTAs, at most 4 per SM, at
    least 1."""
    return max(1, min(-(-n_hint // PROJ_THREADS), PROJ_MIN_CTAS * sm_count))


def project_passes(n_vis: int, grid: int, warp: int = 0) -> int:
    """project.cu:692-696 (project_loop, every projection kernel's loop): grid-stride passes of global warp `warp`.  Warp w
    projects slots [w * 32 + p * stride, + 32) in pass p, stride = grid * 128; warp 0 takes the most passes, the last
    warp of the grid the fewest."""
    r0 = warp * 32
    return 0 if r0 >= n_vis else -(-(n_vis - r0) // (grid * PROJ_THREADS))


def project_min_passes(n_vis: int, grid: int) -> int:
    """The passes of the grid's last warp: every warp of the launch strides at least this often."""
    return project_passes(n_vis, grid, grid * PROJ_WARPS - 1)


def project_warp_slots(n_vis: int, grid: int, warp: int, p: int) -> range:
    """The slots (records) global warp `warp` projects in pass p."""
    r0 = warp * 32 + p * grid * PROJ_THREADS
    return range(min(r0, n_vis), min(r0 + 32, n_vis))


def splat_depth_grid(n_hint: int, sm_count: int = H100_SMS) -> int:
    """scene_depth.cu:47, 53 (launch_splat_depth, launch_splat_depth_scene) through entry_src.cuh:114-119
    (persistent_grid): ceil(n_hint / 256) CTAs, at most 8 per SM, at least 1."""
    return max(1, min(-(-n_hint // SD_THREADS), SD_CTAS_PER_SM * sm_count))


def splat_depth_passes(n_vis: int, grid: int) -> int:
    """scene_depth.cu:19 (splat_depth_body): grid-stride passes of thread 0 (the most any thread takes)."""
    return -(-n_vis // (grid * SD_THREADS))


def scene_keygen_grid(queued: bool, sm_count: int = H100_SMS, kg_ctas_per_sm_fit: int = COOP_CTAS_PER_SM,
                      scene_ctas_per_sm_fit: int = COOP_CTAS_PER_SM) -> int:
    """api.cu:271-276, 489 (bgs_context_create kg_grid / kg_grid_async, enqueue_frame): keygen_scene_kernel's CTAs, the
    single-cloud key-gen grid capped by the scene kernel's own occupancy (`scene_ctas_per_sm_fit`, kg_scene_per_sm).
    Queued frames run exactly sm_count CTAs (both occupancies are at least 1); a synchronous frame at most 4 per SM,
    whatever the occupancies are."""
    return min(coop_grid(sm_count, kg_ctas_per_sm_fit, queued), sm_count * scene_ctas_per_sm_fit)


def keygen_cta_tiles(n: int, grid: int) -> list[tuple[int, int]]:
    """keygen.cu:71: the [t0, t1) range of 2048-gaussian tiles each key-gen CTA owns (phase 1 walks them in order,
    phase 2 expands their mask words in chunks of KG_CHUNK_TILES tiles)."""
    tiles = -(-n // KG_TILE)
    return [(b * tiles // grid, (b + 1) * tiles // grid) for b in range(grid)]


BIN_VIEWS_CTAS_PER_SM_FIT = 3    # bin.cu:328-331: bin_emit_views_kernel's own occupancy (80 registers x 256 threads)
DRV_THREADS, DRV_CTAS_PER_SM = 256, 4   # project.cu:1055: depth_range_views_kernel's CTA size and its cap per SM


def views_tiles(sizes) -> list[int]:
    """api.cu:945-950 (render_entities_impl, vt.tile0): each view's tile0, then the total (tile0[v]); `sizes` are the
    views' (width, height)."""
    out = [0]
    for w, h in sizes:
        out.append(out[-1] + num_tiles(w, h))
    return out


def views_bin_grid(sm_count: int, queued: bool, views_per_sm: int = BIN_VIEWS_CTAS_PER_SM_FIT) -> int:
    """bin.cu:327-333 (launch_bin_emit_views): the binning grid planned for bin_emit_coop_kernel, capped by the views
    kernel's own co-resident CTAs."""
    return min(bin_grid(sm_count, queued), views_per_sm * sm_count)


def depth_range_views_grid(n_hint: int, sm_count: int = H100_SMS) -> int:
    """project.cu:1198-1202 (launch_depth_range_views) through entry_src.cuh:114-119 (persistent_grid): ceil(n_hint / 256)
    CTAs, at most 4 per SM, at least 1."""
    return max(1, min(-(-n_hint // DRV_THREADS), DRV_CTAS_PER_SM * sm_count))


def depth_range_views_passes(n_vis: int, grid: int) -> int:
    """project.cu:1106 (depth_range_views_kernel's pass): grid-stride passes of CTA 0 (the most any CTA takes)."""
    return -(-n_vis // (grid * DRV_THREADS))


def depth_range_views_cta(p: int, grid: int) -> int:
    """project.cu:1106: the CTA whose pass reads sorted position p."""
    return (p // DRV_THREADS) % grid


def warp_first_miss_rounds(length: int, first: int) -> int:
    """project.cu:1076-1091 (warp_first_miss): the rounds of the 32-way search over [0, length) whose first miss is at
    `first` (length when there is none)."""
    lo, hi, rounds = 0, length, 0
    while lo < hi:
        rounds += 1
        step = (hi - lo + 31) // 32
        f = next((lane for lane in range(32) if lo + lane * step >= hi or lo + lane * step >= first), None)
        if f is None:
            lo += 31 * step + 1
        else:
            hi = min(hi, lo + f * step)
            if f > 0:
                lo += (f - 1) * step + 1
    assert lo == first
    return rounds


def device_sm_count(device: int = 0) -> int:
    import torch

    return torch.cuda.get_device_properties(device).multi_processor_count
