"""Inputs and shared checks of tests/test_gpu_views_scale.py: views frames (bgs_render_views, bgs_render_views_aux) large
enough to leave the small-frame paths of binning, the tile-id sort, key-gen and the per-view Depth range.

* A  tile-id sort passes: view sets of exactly 256, 257, 65 536 and 65 537 tiles, and 9 x 1920x1080 (73 440 tiles),
     with a 65535 x 17 view (tiles_x = 4096) between 1080p views.
* B  footprint classes: five views of tiles_x 1, 31, 32, 33 and 120, each with tiny, medium and large footprints, with
     few or many large ones (large_split_parts 16 and 1).
* C  multi-sub-tile binning: 8 views of a 130 000-gaussian room, more visible entries than the binning grid x 2048.
* D  multi-chunk key-gen over the v k segments: 64 views x 1 entity and 8 views x 8 entities, v N > 132 x 16 x 2048.
* E  many views: 64 views of mixed sizes (1x1, 16x16, 17x17, ...) and 32 views x 2 entities, a view that sees nothing.
* F  starved grids: the views frames after a frame of one visible entry.
* G  the per-view Depth range: views with long visible runs, all, one and no visible entries, first two positions in
     different CTAs.
* H  the pair-list overflow frame of test_gpu_views, against its views' own frames.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

import bevy_gaussian_splatting_b200 as B
import entity_cases as E
import kernel_paths as KP
import scene_cases as SC
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import entity_settings

f32 = np.float32
ROOM = (0.0, 1.5, -1.0)
FORMATS = {"f32": (np.float32, torch.float32, abi.BGS_FORMAT_RGBA32F), "f16": (np.float16, torch.float16, abi.BGS_FORMAT_RGBA16F),
           "u8": (np.uint8, torch.uint8, abi.BGS_FORMAT_RGBA8_SRGB)}


# ---------------------------------------------------------------------------------------------------------------------
# targets, calls and hooks

def ok(p, rc):
    assert rc == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)


def target(view, fmt, device):
    npd, tod, _ = FORMATS[fmt]
    if device:
        return torch.empty((view.height, view.width, 4), dtype=tod, device="cuda")
    return np.empty((view.height, view.width, 4), npd)


def addr(t):
    return t.data_ptr() if isinstance(t, torch.Tensor) else t.ctypes.data


def as_bytes(t):
    if isinstance(t, torch.Tensor):
        torch.cuda.synchronize()
        return t.cpu().numpy().tobytes()
    return t.tobytes()


def as_host(t):
    if isinstance(t, torch.Tensor):
        torch.cuda.synchronize()
        return t.cpu().numpy()
    return t


def depth_buffer(view, seed):
    """A per-view depth buffer (about half a room's splats lie behind it somewhere)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand((view.height, view.width), generator=g, device="cuda") * 0.04


class Scene:
    """An entity list on a context: the arguments of its views, views_aux, entities_ex and entities_aux calls.
    `listed`: [(cloud, layout, transform, CloudSettings)]."""

    def __init__(self, p, listed, bits=None, frame_box=False):
        self.p = p
        up = {}
        self.handles, self.unis, self.sts, self.oracle = [], [], [], []
        for cloud, layout, tr, st in listed:
            if id(cloud) not in up:
                up[id(cloud)] = p.add_cloud(cloud, f16=layout in ("f16", "cov"), precompute_covariance=layout == "cov")
            h = up[id(cloud)]
            self.handles.append(h)
            self.unis.append(p.cloud_uniform(st, tr, h.aabb))
            self.sts.append(st)
            self.oracle.append(E.oracle_entry(cloud, layout, self.unis[-1], st))
        self.bits = list(bits) if bits is not None else [0] * len(listed)
        self.frame_box = frame_box
        self.n_view = sum(len(c.position_visibility) for c, _, _, _ in listed)

    def common(self, flags=0):
        k = len(self.handles)
        s = self.sts[0].to_abi()
        s.flags = (s.flags & ~abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX) | flags | (abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX if self.frame_box else 0)
        return ((C.c_void_p * k)(*[h._h.value for h in self.handles]), (abi.bgs_cloud_uniform * k)(*self.unis),
                (abi.bgs_entity_settings * k)(*[entity_settings(st) for st in self.sts]), (C.c_uint32 * k)(*self.bits), k, s)

    def _depths(self, views, depths):
        n = len(views)
        return None if depths is None else (abi.bgs_scene_depth * n)(
            *[abi.bgs_scene_depth(depth=d.data_ptr(), pitch_bytes=4 * v.width) for d, v in zip(depths, views)])

    def views(self, views, outs, fmt, flags=0, depths=None, device=False):
        clouds, unis, es, bits, k, s = self.common(flags)
        n = len(views)
        vs = (abi.bgs_view * n)(*[v.to_abi() for v in views])
        return self.p._lib.bgs_render_views(self.p._ctx, clouds, unis, es, bits, k, vs, n, C.byref(s), self._depths(views, depths),
                                            (C.c_void_p * n)(*[addr(o) for o in outs]), FORMATS[fmt][2], int(device))

    def views_aux(self, views, outs, fmt, flags=0, depths=None, device=False):
        clouds, unis, es, bits, k, s = self.common(flags)
        n = len(views)
        vs = (abi.bgs_view * n)(*[v.to_abi() for v in views])
        tg = [(C.c_void_p * n)(*[addr(o[f]) for o in outs]) for f in range(3)]
        return self.p._lib.bgs_render_views_aux(self.p._ctx, clouds, unis, es, bits, k, vs, n, C.byref(s),
                                                self._depths(views, depths), *tg, FORMATS[fmt][2], int(device))

    def ex(self, view, out, fmt, flags=0, depth=None, device=False):
        clouds, unis, es, bits, k, s = self.common(flags)
        zd = None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * view.width)
        return self.p._lib.bgs_render_entities_ex(self.p._ctx, clouds, unis, es, bits, k, C.byref(view.to_abi()), C.byref(s),
                                                  None, None if zd is None else C.byref(zd), addr(out), FORMATS[fmt][2], int(device))

    def aux(self, view, outs, fmt, flags=0, depth=None, device=False):
        clouds, unis, es, bits, k, s = self.common(flags)
        zd = None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * view.width)
        return self.p._lib.bgs_render_entities_aux(self.p._ctx, clouds, unis, es, bits, k, C.byref(view.to_abi()), C.byref(s),
                                                   None, None if zd is None else C.byref(zd), *[addr(o) for o in outs],
                                                   FORMATS[fmt][2], int(device))

    def oracle_frame(self, view, depth=None):
        """entity_oracle's frame of one view (its depth buffer as a host array, or None)."""
        from entity_oracle import entity_oracle as EO

        return EO.frame(self.oracle, view.to_abi(), [st.to_abi() for st in self.sts], [st.num_classes for st in self.sts],
                        scene=None if depth is None else depth.cpu().numpy(), entity_flags=self.bits)


def hooks(p, depth_tested):
    """Everything the last frame leaves readable, as arrays."""
    torch.cuda.synchronize()
    rec, ids = p.projected()
    got = dict(stats=p.frame_stats(), sorted=p.sorted_entries(), records=rec, ids=ids, ranges=p.tile_ranges(),
               entries=p.tile_entries())
    got["splat_depths"] = p.splat_depths() if depth_tested else None
    return got


def check_restricted(got, wants, views):
    """The joint frame's hooks `got` restricted to view i are view i's one-round single-view hooks wants[i]: view i's
    entries are the global indices [i n, (i + 1) n), that subsequence of the sorted entries, records, ids and splat depths
    is view i's, and view i's block of tile ranges gives the same lengths and, through the ids, the same entries."""
    n = got["stats"].n // len(views)
    assert got["stats"].n == n * len(views) and got["stats"].rounds == 1 and got["stats"].tiles_y == 1
    assert (got["stats"].width, got["stats"].height) == (views[0].width, views[0].height)
    tile0 = n_vis = n_pairs = 0
    srt = got["sorted"]
    for i, (v, want) in enumerate(zip(views, wants)):
        n_vis += want["stats"].n_visible
        n_pairs += want["stats"].n_pairs
        mine = (srt[:, 1] >= i * n) & (srt[:, 1] < (i + 1) * n)
        sub = srt[mine].copy()
        sub[:, 1] -= i * n
        assert np.array_equal(sub, want["sorted"]), ("sorted", i)
        rmine = (got["ids"] >= i * n) & (got["ids"] < (i + 1) * n)
        assert got["records"][rmine].tobytes() == want["records"].tobytes(), ("records", i)
        assert np.array_equal(got["ids"][rmine] - i * n, want["ids"]), ("ids", i)
        if want["splat_depths"] is not None:
            assert got["splat_depths"][rmine].tobytes() == want["splat_depths"].tobytes(), ("splat depths", i)
        tiles = KP.num_tiles(v.width, v.height)
        block = got["ranges"][tile0:tile0 + tiles].astype(np.int64)
        wr = want["ranges"].astype(np.int64)
        assert np.array_equal(block[:, 1] - block[:, 0], wr[:, 1] - wr[:, 0]), ("ranges", i)
        # (all of the block's entries at once: each tile's slice, in tile order, is the concatenation)
        g = np.concatenate([got["entries"][a:b] for a, b in block]) if tiles else np.zeros(0, np.uint32)
        w = np.concatenate([want["entries"][a:b] for a, b in wr]) if tiles else np.zeros(0, np.uint32)
        assert np.array_equal(got["ids"][g].astype(np.int64) - i * n, want["ids"][w].astype(np.int64)), ("tile entries", i)
        tile0 += tiles
    assert tile0 == got["stats"].tiles_x
    assert (got["stats"].n_visible, got["stats"].n_pairs) == (n_vis, n_pairs)


def check_oracle(want_hooks, image, orc, tol=1e-3):
    """A single-view frame's hooks and pixels against entity_oracle's frame of that view: sorted entries, n_vis, n_pairs,
    rank_to_id, tile ranges and tile entries bit for bit, pixels within tol."""
    fs = want_hooks["stats"]
    assert (fs.n_visible, fs.n_pairs) == (orc["n_vis"], orc["n_pairs"])
    assert np.array_equal(want_hooks["sorted"], orc["sorted"]), "sorted entries differ from the oracle's"
    assert np.array_equal(want_hooks["ids"], orc["rank_to_id"]), "rank_to_id differs from the oracle's"
    assert np.array_equal(want_hooks["ranges"], orc["tile_ranges"]), "tile ranges differ from the oracle's"
    assert np.array_equal(want_hooks["entries"], orc["tile_entries"]), "tile entries differ from the oracle's"
    if image is not None:
        assert float(np.abs(as_host(image).astype(np.float64) - orc["image"]).max()) <= tol


def footprint_counts(records, ids, n_view, v):
    """Per view, {class: count} of the joint frame's records (bin.cu's classes, from each record's bbox)."""
    bb = records[:, 6:8].view(np.uint32)
    xlo, xhi, ylo, yhi = bb[:, 0] & 0xFFFF, bb[:, 0] >> 16, bb[:, 1] & 0xFFFF, bb[:, 1] >> 16
    drawn = (xlo <= xhi) & (ylo <= yhi)
    tiles = np.where(drawn, (xhi // 16 - xlo // 16 + 1) * (yhi // 16 - ylo // 16 + 1), 0).astype(np.int64)
    view = ids.astype(np.int64) // n_view
    out = []
    for i in range(v):
        t = tiles[view == i]
        out.append({"tiny": int(((t > 0) & (t <= KP.BIN_TINY)).sum()), "medium": int(((t > KP.BIN_TINY) & (t <= KP.BIN_BIG)).sum()),
                    "large": int((t > KP.BIN_BIG).sum())})
    return out


# ---------------------------------------------------------------------------------------------------------------------
# clouds and entity lists

def room_cloud(n, seed, sh_degree=1, half=1.2, scale=0.08):
    return SC.cloud_in_box(n, seed, centre=ROOM, half=half, scale=scale, sh_degree=sh_degree)


def quad_entities(cloud, scale=1.0):
    """Two quad-uv 3DGS entities of one cloud (raster_kernel<0, ...>'s MODE 0 loop in a views frame)."""
    return [(cloud, "f32", SC.transform(), B.CloudSettings(global_scale=scale)),
            (cloud, "f32", SC.transform((0.3, -0.1, 0.2), 0.9, 0.5), B.CloudSettings(global_scale=0.8 * scale, global_opacity=0.8))]


def mixed_entities(cloud, scale=1.0):
    """A quad-uv and a conic entity (raster_kernel<3, ...>)."""
    return [(cloud, "f32", SC.transform(), B.CloudSettings(global_scale=scale)),
            (cloud, "f32", SC.transform((-0.2, 0.1, 0.3), 1.1, -0.4), B.CloudSettings(global_scale=scale, aabb=True))]


def around(i, count, w, h, radius=3.5, fov=math.pi / 4, height=0.3):
    """Camera i of `count` on an arc in front of the room, looking at its centre."""
    a = -0.9 + 1.8 * i / max(count - 1, 1)
    eye = (ROOM[0] + radius * math.sin(a), ROOM[1] + height * math.cos(3 * a), ROOM[2] + radius * math.cos(a))
    return B.perspective_view(eye, ROOM, w, h, fov_y=fov)


def _fov_for(h, focal=1000.0):
    return 2.0 * math.atan(h / (2.0 * focal))


# ---- A: tile totals
WIDE = (65535, 17)       # tiles_x = 4096, tiles_y = 2: 8192 tiles
HD = (1920, 1080)        # 8160 tiles
TILE_SETS = {
    "t256": [(160, 160), (200, 120), (200, 60)],
    "t257": [(160, 160), (1, 1), (200, 120), (200, 60)],
    "t65536": [HD, WIDE, HD, HD, (2096, 1024), HD, HD, HD],
    "t65537": [HD, WIDE, HD, HD, (2096, 1024), HD, HD, HD, (1, 1)],
    "t9x1080": [HD] * 9,
}
TILE_TOTALS = {"t256": 256, "t257": 257, "t65536": 65536, "t65537": 65537, "t9x1080": 73440}
TILE_PASSES = {"t256": 1, "t257": 2, "t65536": 2, "t65537": 3, "t9x1080": 3}


def tile_set(name):
    sizes = TILE_SETS[name]
    out = []
    for i, (w, h) in enumerate(sizes):
        # the wide strip: a narrow vertical field through the room's middle; the 1x1 views: straight at the centre
        fov = 0.02 if (w, h) == WIDE else (math.pi / 3 if (w, h) == (1, 1) else math.pi / 4)
        out.append(around(i, len(sizes), w, h, fov=fov, height=0.0 if h <= 17 else 0.3))
    return out


# ---- B: footprint classes
# focal length 1000 px in every view (fov from the height): a gaussian's footprint depends on its scale / distance only
B_SIZES = [(16, 2176), (496, 400), (512, 300), (528, 500), (1920, 1080)]   # tiles_x 1, 31, 32, 33, 120
B_N = 6000


def footprint_cloud(n_large, seed=3):
    """B_N gaussians in a small box at the room's centre, a third each tiny (scale 0.0012), medium (0.012) and of
    every size between, and n_large giants (scale 1.5, opacity 0.03) on the vertical through the centre (inside even the
    16-pixel-wide view's frustum) that are large footprints in every view."""
    rng = np.random.default_rng(seed)
    n = B_N + n_large
    c = B.random_gaussians_3d_seeded(n, seed, sh_degree=0)
    pos = c.position_visibility.copy()
    pos[:, :3] = rng.uniform(-0.25, 0.25, (n, 3)).astype(f32) + np.asarray(ROOM, f32)
    pos[:, 3] = 1.0
    so = c.scale_opacity.copy()
    band = np.arange(n) % 3
    s = np.where(band == 0, 0.0012, np.where(band == 1, 0.012, np.exp(rng.uniform(np.log(0.001), np.log(0.012), n))))
    s[B_N:] = 1.5
    pos[B_N:, 0], pos[B_N:, 2] = ROOM[0], ROOM[2]
    so[:, :3] = (s[:, None] * rng.uniform(0.8, 1.0, (n, 3))).astype(f32)
    so[:, 3] = np.where(np.arange(n) < B_N, np.maximum(so[:, 3], 0.4), 0.03).astype(f32)
    return B.PlanarGaussian3d(pos, c.spherical_harmonic, c.rotation, so)


def footprint_views():
    out = []
    for i, (w, h) in enumerate(B_SIZES):
        a = -0.8 + 0.4 * i
        eye = (ROOM[0] + 3.0 * math.sin(a), ROOM[1] + 0.2, ROOM[2] + 3.0 * math.cos(a))
        out.append(B.perspective_view(eye, ROOM, w, h, fov_y=_fov_for(h)))
    return out


# ---- C: multi-sub-tile binning
C_N = 130_000
C_SIZES = [(320, 240), (256, 256), (200, 150), (333, 177), (128, 96), (400, 300), (97, 61), (240, 320)]


def multi_subtile_views():
    return [around(i, len(C_SIZES), w, h, radius=4.5) for i, (w, h) in enumerate(C_SIZES)]


# ---- D / E: many views
D_N = 70_000               # 64 x 70 000 = 4 480 000 > 132 x 16 x 2048 = 4 325 376
D_N8 = 70_000              # 8 views x 8 entities x 70 000
E_SIZES = [(1, 1), (16, 16), (17, 17), (33, 20), (48, 31), (64, 64), (5, 90), (100, 7)]


def many_views(v):
    """v views cycling over E_SIZES, on two arcs around the room; view 5 looks away from it (sees nothing)."""
    out = []
    for i in range(v):
        w, h = E_SIZES[i % len(E_SIZES)]
        a = 2.0 * math.pi * i / v
        r = 3.5 + 0.5 * (i % 3)
        eye = (ROOM[0] + r * math.sin(a), ROOM[1] + 0.4 * math.cos(2 * a), ROOM[2] + r * math.cos(a))
        tgt = ROOM if i != 5 else tuple(2 * e - c for e, c in zip(eye, ROOM))
        out.append(B.perspective_view(eye, tgt, w, h, fov_y=math.pi / 4 if w * h > 1 else math.pi / 3))
    return out


def eight_entities(cloud):
    """8 entities of one cloud, each its own transform, scale and kind (quad-uv or conic): 64 segments over 8 views."""
    out = []
    for j in range(8):
        st = B.CloudSettings(global_scale=0.8 + 0.05 * j, global_opacity=1.0 - 0.05 * j, aabb=j % 3 == 2)
        out.append((cloud, "f32", SC.transform((0.05 * (j - 4), 0.02 * (j % 3), -0.03 * (j % 2)), 0.9 + 0.02 * j, 0.2 * j), st))
    return out


# ---- F: starved grids
def starve_cloud():
    """One small gaussian on the starving view's axis (stride_cases.starve_cloud)."""
    return B.PlanarGaussian3d(np.array([[0.0, 1.5, 0.0, 1.0]], f32), np.zeros((1, 48), f32),
                              np.array([[1.0, 0.0, 0.0, 0.0]], f32), np.array([[0.01, 0.01, 0.01, 0.5]], f32))


STARVE_VIEW = B.headless_view(256, 192)
F_N = 30_000
F_SIZES = [(320, 240), (200, 120), (97, 61), (256, 192), (33, 250), (160, 160)]


def stride_views():
    return [around(i, len(F_SIZES), w, h) for i, (w, h) in enumerate(F_SIZES)]


# ---- G: the per-view Depth range
G_NEAR = 6000                    # gaussians in a small box at the origin
G_FIRST_MISS = 2500              # index of the marker at (20, 0, 0): the near views' first culled index
G_LAST_MISS = G_NEAR - 1 - 2200  # index of the marker at (-20, 0, 0): their last culled index
G_FAR_MISS = 4000                # index of the marker at (20, 20, -57)
MARKERS = {G_FIRST_MISS: (20.0, 0.0, 0.0), G_LAST_MISS: (-20.0, 0.0, 0.0), G_FAR_MISS: (20.0, 20.0, -57.0)}


def depth_range_cloud(seed=5):
    c = B.random_gaussians_3d_seeded(G_NEAR, seed, sh_degree=0)
    pos = c.position_visibility.copy()
    pos[:, :3] = pos[:, :3] * f32(0.3 / 20.0)
    for i, xyz in MARKERS.items():
        pos[i, :3] = xyz
    pos[:, 3] = 1.0
    so = c.scale_opacity.copy()
    so[:, :3] *= f32(0.05)
    so[:, 3] = np.maximum(so[:, 3], 0.5)
    return B.PlanarGaussian3d(pos, c.spherical_harmonic, c.rotation, so)


def depth_range_views(w=64, h=48):
    """name -> view.  near*: the box, not the markers at (+-20, 0, 0); all: everything; one: only (20, 0, 0); two: (20, 0, 0)
    at depth ~3 and (20, 20, -57) at depth ~63 (so its first two sorted positions lie thousands apart); none: nothing."""
    return {
        "near0": B.perspective_view((0.0, 0.0, 5.0), (0.0, 0.0, 0.0), w, h),
        "all": B.perspective_view((0.0, 0.0, 60.0), (0.0, 0.0, 0.0), w, h),
        "near1": B.perspective_view((1.0, 1.5, 4.5), (0.0, 0.0, 0.0), w + 30, h + 7),
        "one": B.perspective_view((20.0, 0.0, 3.0), (20.0, 0.0, 0.0), w, h, fov_y=math.pi / 8),
        "two": B.perspective_view((20.0, 0.0, 3.0), (20.0, 10.0, -27.0), w, h, fov_y=math.pi / 2),
        "none": B.perspective_view((0.0, 0.0, 5.0), (0.0, 0.0, 10.0), w, h),
        "near2": B.perspective_view((-2.0, -1.0, 4.0), (0.0, 0.0, 0.0), 33, 250),
    }


def visible_run(sorted_entries, n_vis_total, i, n):
    """View i's visible global indices in ascending order (the stable compaction's run) from the joint sorted entries."""
    g = np.sort(sorted_entries[:n_vis_total, 1].astype(np.int64))
    return g[(g >= i * n) & (g < (i + 1) * n)] - i * n


def first_misses(run, n):
    """(first culled index, last culled index counted from the back) of a view's visible run of n entries: where the
    run first departs from 0, 1, ... and, read backwards, from n - 1, n - 2, ...; len(run) when it never does."""
    cnt = len(run)
    fwd = np.nonzero(run != np.arange(cnt))[0]
    bwd = np.nonzero(run[::-1] != n - 1 - np.arange(cnt))[0]
    return (int(fwd[0]) if len(fwd) else cnt), (int(bwd[0]) if len(bwd) else cnt)
