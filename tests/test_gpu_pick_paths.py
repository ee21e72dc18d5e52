"""bgs_render_entities_pick on the H100 where bgs_render_entities_ex does not run the generic blend loop a pick frame runs.

- Colour identity.  On homogeneous entity lists (3DGS and 2DGS quad-uv, 3DGS conic, 2DGS surfel) of 1, 2 and 5 entities,
  in every layout, the pick frame's colour is bgs_render_entities_ex's byte for byte, made with the same flags, whichever
  path the latter takes: for quad-uv lists raster_kernel<0, false>'s inline-asm loop, raster2_kernel<false, Z> after a
  frame of large footprints, and binning rounds through raster2_kernel<true, Z> under BGS_FLAG_CHUNKS (each path asserted
  through kernel_paths).  Its hooks and stats are the one-round frame's, its depths the splat depths bit for bit.
- Exact ties.  Splats on the view axis of an odd viewport are centred on a pixel centre, where every kind's coverage
  exponent is exactly 0: the weights are restated exactly in f32, and equal weights must go to the pair earlier in blend
  order, also when that pair belongs to the later entity.
- Record mapping.  64 entities, clouds of 1 .. 4097 gaussians in several layouts, one cloud listed many times: the first
  and last gaussian of every entity alone on its own tile, each picked exactly.
Runtime on an H100: about 35 s for the file."""
import numpy as np
import pytest
import torch

import bevy_gaussian_splatting_b200 as B
import kernel_paths as KP
import pick_cases as PK
import scene_cases as SC
import scene4d_cases as S4
from bevy_gaussian_splatting_b200 import abi
from entity_oracle import entity_oracle as EO

pytestmark = pytest.mark.gpu

f32 = np.float32
G = B.GaussianMode
W, H = 200, 120   # (not tile multiples)
VIEW = B.headless_view(W, H)

KINDS = {"3dgs_obb": dict(), "2dgs_obb": dict(gaussian_mode=G.Gaussian2d), "3dgs_aabb": dict(aabb=True),
         "2dgs_aabb": dict(gaussian_mode=G.Gaussian2d, aabb=True)}
# MODE 0 (quad-uv) lists: the path bgs_render_entities_ex takes; the others always run the generic loop
PATHS = {"3dgs_obb": ("one_round", "raster2", "rounds"), "2dgs_obb": ("one_round", "raster2", "rounds"),
         "3dgs_aabb": ("generic",), "2dgs_aabb": ("generic",)}
CASES = [(kind, n, path) for kind in KINDS for n in (1, 2, 5) for path in PATHS[kind]]
LARGE_SCALE = 6.0   # global_scale of the raster2 lists: >= 8 pairs per visible splat


def entity_list(kind, n, large=False):
    """[(cloud, layout, transform, CloudSettings)]: n entities of one blend kind over the room's clouds (f32 SH 3, f16 SH 1,
    covariance, f32 SH 0; 2DGS lists leave out the covariance cloud, which has no rotation), one cloud always listed twice
    with different transforms when n > 1."""
    room = S4.room()
    layouts = [room[0], room[1], room[3]] if kind.startswith("2dgs") else room
    over = dict(KINDS[kind], global_scale=LARGE_SCALE) if large else KINDS[kind]
    out = []
    for j in range(n):
        cloud, layout, _, tr, kw = layouts[j % len(layouts)] if j < n - 1 or n == 1 else layouts[0]
        if j == n - 1 and n > 1:   # the first cloud again, moved and turned
            tr = SC.transform((0.3, -0.2, 0.5), 0.9, 0.6)
        out.append((cloud, layout, tr, B.CloudSettings(**{**kw, **over})))
    return out


def _depth(seed):
    return torch.rand((H, W), generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda") * 0.04


@pytest.mark.parametrize("with_depth", [False, True])
@pytest.mark.parametrize("kind,n,path", CASES)
def test_pick_colour_is_entities_ex_on_every_path(kind, n, path, with_depth):
    listed = entity_list(kind, n, large=path == "raster2")
    depth = _depth(11) if with_depth else None
    chunk_flag = abi.BGS_FLAG_CHUNKS if path == "rounds" else abi.BGS_FLAG_NO_CHUNKS
    p = B.GaussianSplattingPlugin(0)   # (a fresh context: no hints from another test's frames)
    try:
        sc = PK.Scene(p, listed, [0] * n, VIEW)
        rng = np.random.default_rng(7)
        for fmt in PK.FORMATS:
            for device in (False, True):
                for mode, mflag in PK.MODES.items():
                    if mode == "over" and not device:
                        continue   # (host blend-over reads the context's last frame: covered by the device target)
                    flags = mflag | chunk_flag
                    fill = None
                    if mode == "over":
                        fill = (rng.random((H, W, 4)) * (255 if fmt == "u8" else 1)).astype(PK.FORMATS[fmt][0])
                    out, pick = PK.target(VIEW, fmt, device, fill), PK.pick_target(VIEW, device)
                    PK.ok(p, sc.call("pick", out, fmt, flags, depth, device, pick))
                    got = PK.hooks(p)
                    sd = p.splat_depths()
                    fs = p.frame_stats()
                    assert fs.rounds == 1
                    # the hints the next frame plans with are this frame's counts
                    assert KP.large_footprint_raster(fs.n_visible, fs.n_pairs) == (path == "raster2"), (fs.n_visible, fs.n_pairs)
                    want = PK.target(VIEW, fmt, device, fill)
                    PK.ok(p, sc.call("ex", want, fmt, flags, depth, device))
                    assert (p.frame_stats().rounds > 1) == (path == "rounds")
                    assert PK.as_bytes(out) == PK.as_bytes(want), (fmt, device, mode)
                    if path == "rounds":   # hooks and stats: the same frame in one round
                        one = PK.target(VIEW, fmt, device, fill)
                        flags1 = (flags & ~abi.BGS_FLAG_CHUNKS) | abi.BGS_FLAG_NO_CHUNKS
                        PK.ok(p, sc.call("ex", one, fmt, flags1, depth, device))
                        assert PK.as_bytes(one) == PK.as_bytes(want), (fmt, device, mode)
                    want_hooks = PK.hooks(p)
                    for key in want_hooks:
                        assert got[key] == want_hooks[key], key
                    pk = PK.pick_host(pick, VIEW)
                    _, ids = p.projected()
                    rank = PK.to_rank(pk, ids, sc.counts)
                    some = rank >= 0
                    assert some.mean() > 0.1
                    assert np.array_equal(pk["depth"][some].view(np.uint32), sd[rank[some]].view(np.uint32))
                    assert (pk["entity"][~some] == abi.BGS_PICK_NONE).all() and (pk["weight"][~some] == 0).all()
    finally:
        p.destroy()


@pytest.mark.parametrize("path", ["raster2", "rounds"])
def test_pick_colour_is_raster2_bytes_at_1080p(path):
    """rgba8 sRGB at 1920 x 1080 through raster2_kernel's own encoder (store_pixel2): millions of channel values, so the
    bytes in the narrow bands where two orders of the same encode round apart are compared too."""
    view = B.headless_view(1920, 1080)
    listed = entity_list("3dgs_obb", 5)
    flags = abi.BGS_FLAG_CHUNKS if path == "rounds" else abi.BGS_FLAG_NO_CHUNKS
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = PK.Scene(p, listed, [0] * 5, view)
        out, pick = PK.target(view, "u8", True), PK.pick_target(view, True)
        PK.ok(p, sc.call("pick", out, "u8", flags, None, True, pick))
        fs = p.frame_stats()
        assert KP.large_footprint_raster(fs.n_visible, fs.n_pairs), (fs.n_visible, fs.n_pairs)
        want = PK.target(view, "u8", True)
        PK.ok(p, sc.call("ex", want, "u8", flags, None, True))
        assert (p.frame_stats().rounds > 1) == (path == "rounds")
        assert torch.equal(out, want)
    finally:
        p.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# exact ties.  On the view axis of a 63 x 47 viewport a splat's centre is (31.5, 23.5), pixel (31, 23)'s centre, so its
# coverage exponent there is 0 for every kind: ex2.approx(0) (quad-uv), __expf(0) (conic), power = -0 (surfel), and
# a = min(opacity, 0.999) exactly.  The pixel's pairs then blend with w = a T and T = fmaf(-a, T, T), restated below in f32.

TW, TH = 63, 47
TVIEW = B.headless_view(TW, TH)
CX, CY = TW // 2, TH // 2
TIE_KINDS = {"quad": dict(), "quad_2d": dict(gaussian_mode=G.Gaussian2d), "conic": dict(aabb=True),
             "surfel": dict(gaussian_mode=G.Gaussian2d, aabb=True)}
TIE_LAYOUTS = ("f32", "f16", "cov", "sh0")
CULLED_Z = 9.0   # (behind the camera at z = 5: culled, but part of the index space)


def _tie_cloud(zs, opacities, at, layout, xs=None, scale=0.05):
    """A cloud of len(at) + 2 gaussians: gaussian at[i] at (xs[i] or 0, 1.5, zs[i]) with opacities[i], the rest culled.
    The gaussians are anisotropic and turned: an isotropic 3DGS splat seen head-on has a circular footprint, whose quad
    axes the projection leaves NaN (the oracle's too), so it covers no pixel."""
    n = max(at) + 2
    pos = np.tile(np.array([0.0, 1.5, CULLED_Z, 1.0], f32), (n, 1))
    so = np.tile(np.array([1.3 * scale, scale, 0.8 * scale, 0.5], f32), (n, 1))
    for k, i in enumerate(at):
        pos[i, 0] = 0.0 if xs is None else xs[k]
        pos[i, 2] = zs[k]
        so[i, 3] = opacities[k]
    rng = np.random.default_rng(n)
    sh = rng.uniform(-0.5, 0.5, (n, 48)).astype(f32)
    q = np.array([0.9, 0.1, 0.2, 0.3], f32)
    rot = np.tile(q / np.linalg.norm(q), (n, 1)).astype(f32)
    c = B.PlanarGaussian3d(pos, sh, rot, so)
    return c.with_sh_degree(0) if layout == "sh0" else c


def _fma(a, b, c):
    """fmaf in f32: the f64 product of two f32 values is exact, and so is the sum here (|c| >= |a b|), so one rounding."""
    return f32(float(a) * float(b) + float(c))


def _restate(opacities):
    """The f32 weights of pairs blending front to back at a pixel where every exponent is 0."""
    T, ws = f32(1.0), []
    for o in opacities:
        a = min(f32(o), f32(0.999))
        ws.append(f32(a * T))
        T = _fma(-a, T, T)
    return ws


def _tie_scene(case, layout):
    """(listed, entity flags, expected (entity, index), expected weight): entity 1's pair is in front of entity 0's."""
    lay = "f32" if layout == "sh0" else layout
    if case == "thirds":       # 0.25 then f32(1/3): both weights exactly 0.25
        front = _tie_cloud([1.0], [0.25], [2], layout)
        back = _tie_cloud([0.0], [f32(1.0) / f32(3.0)], [1], layout)
        return [(back, lay, None), (front, lay, None)], [0, 0], (1, 2), [0.25, f32(1.0) / f32(3.0)]
    if case == "zeros":        # a stack of zero-opacity splats: every w is +0, the front-most is picked
        a = _tie_cloud([0.5, -0.5], [0.0, 0.0], [0, 3], layout)
        b = _tie_cloud([1.0, 0.0], [0.0, 0.0], [1, 2], layout)
        # blend order: b[1] (z 1.0), a[0] (z 0.5), b[2] (z 0), a[3] (z -0.5)
        return [(a, lay, None), (b, lay, None)], [0, 0], (1, 1), [0.0, 0.0, 0.0, 0.0]
    # "edge": a front splat of opacity 0.5, behind it entity 0 with its overlay, whose edge band covers the pixel: w = T = 0.5
    front = _tie_cloud([1.0], [0.5], [1], layout)
    back = _tie_cloud([0.0], [0.9], [0], layout)
    return [(back, lay, "edge"), (front, lay, None)], [1, 0], (1, 1), [0.5]


def _edge_offset(cloud, layout, st):
    """An x offset of gaussian 0 of `cloud` that puts pixel (CX, CY) on its quad's edge band, found with the entity
    oracle (the same records and decisions, bit for bit)."""
    for dx in np.linspace(0.02, 0.6, 59):
        c = B.PlanarGaussian3d(cloud.position_visibility.copy(), cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity)
        c.position_visibility[0, 0] = f32(dx)
        u = B.GaussianSplattingPlugin.cloud_uniform(st)
        fr = EO.frame([(SC.oracle_cloud(c, layout), u, layout == "cov")], TVIEW.to_abi(), [st.to_abi()], [1],
                      entity_flags=[1])
        if fr["edge_mask"][CY, CX]:
            return c
    raise AssertionError("no offset puts the pixel on the edge band")


# (f16 opacities: two pairs of dyadic alphas a1, a2 < 1 never tie exactly, a1 = a2 (1 - a1) has no such solution; the
# covariance layout is 3DGS only)
TIE_CASES = [(case, kind, layout) for case in ("thirds", "zeros", "edge") for kind in TIE_KINDS for layout in TIE_LAYOUTS
             if not (case == "thirds" and layout in ("f16", "cov")) and not (layout == "cov" and kind in ("quad_2d", "surfel"))]


@pytest.mark.parametrize("case,kind,layout", TIE_CASES)
def test_exact_ties_go_to_the_earlier_pair(case, kind, layout):
    specs, flags, (want_e, want_i), ops = _tie_scene(case, layout)
    st = B.CloudSettings(**TIE_KINDS[kind], opacity_adaptive_radius=False)
    listed = []
    for cloud, lay, role in specs:
        if role == "edge":
            cloud = _edge_offset(cloud, lay, st)
        listed.append((cloud, lay, None, st))
    if layout in ("f16", "cov"):
        ops = [f32(np.float16(o)) for o in ops]
    ws = _restate(ops)
    if case == "edge":
        ws = [ws[0], _fma(-ws[0], f32(1.0), f32(1.0))]   # the edge pair behind it: w = T
    assert all(w.view(np.uint32) == ws[0].view(np.uint32) for w in ws), ws   # a tie, exactly
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = PK.Scene(p, listed, flags, TVIEW)
        for device in (False, True):
            out, pick = PK.target(TVIEW, "f32", device), PK.pick_target(TVIEW, device)
            PK.ok(p, sc.call("pick", out, "f32", 0, None, device, pick))
            rec, ids = p.projected()
            on_axis = rec[:, 0] == f32(TW / 2)
            assert on_axis.sum() == (4 if case == "zeros" else 2 if case == "thirds" else 1)
            assert (rec[on_axis, 1] == f32(TH / 2)).all()
            pk = PK.pick_host(pick, TVIEW)[CY, CX]
            assert (int(pk["entity"]), int(pk["index"])) == (want_e, want_i), (pk, case, kind, layout)
            assert pk["weight"].view(np.uint32) == ws[0].view(np.uint32), (pk["weight"], ws[0])
            g = int(np.cumsum([0] + sc.counts)[want_e]) + want_i
            r = int(np.flatnonzero(ids == g)[0])
            assert pk["depth"].view(np.uint32) == p.splat_depths()[r].view(np.uint32)
    finally:
        p.destroy()


# ---------------------------------------------------------------------------------------------------------------------
# the record mapping at 64 entities: the binary search over the segment offsets, at every segment start and end

MW, MH = 256, 128        # 16 x 8 tiles: entity j's gaussians 0 and n_j - 1 on tiles (2 (j % 8) + {0, 1}, j // 8)
MVIEW = B.headless_view(MW, MH)
MAP_DEPTH = 3.0          # (distance from the camera)


def _world(px, py, d=MAP_DEPTH):
    """The world point at distance d along the camera's -z whose projection is near pixel position (px, py)."""
    t, aspect = np.tan(np.pi / 8), MW / MH
    ndc_x, ndc_y = (px - MW / 2) / (MW / 2), (MH / 2 - py) / (MH / 2)
    return np.array([ndc_x * d * t * aspect, 1.5 + ndc_y * d * t, 5.0 - d], f32)


def _map_cloud(n, layout, seed):
    """n gaussians: 0 at the origin, n - 1 one tile (16 px) to its right at MAP_DEPTH, the others culled."""
    pos = np.tile(np.array([0.0, 0.0, CULLED_Z, 1.0], f32), (n, 1))
    pos[0, :3] = 0.0
    if n > 1:
        pos[n - 1, :3] = _world(MW / 2 + 16, MH / 2) - _world(MW / 2, MH / 2)
    rng = np.random.default_rng(seed)
    so = np.tile(np.array([0.01, 0.01, 0.01, 0.8], f32), (n, 1))
    sh = rng.uniform(-0.5, 0.5, (n, 48)).astype(f32)
    rot = np.tile(np.array([1, 0, 0, 0], f32), (n, 1))
    c = B.PlanarGaussian3d(pos, sh, rot, so)
    return c.with_sh_degree(0) if layout == "sh0" else c


MAP_CLOUDS = [(1, "f32"), (2, "f16"), (31, "cov"), (32, "sh0"), (33, "f32"), (3000, "f16"), (4097, "f32")]


def test_pick_maps_records_at_64_entities():
    clouds = [(_map_cloud(n, lay, s), "f32" if lay == "sh0" else lay) for s, (n, lay) in enumerate(MAP_CLOUDS)]
    listed = []
    for j in range(64):
        # the first seven entities list each cloud once; then the 33-gaussian cloud and the others alternate
        cloud, lay = clouds[j] if j < len(clouds) else clouds[4 if j % 2 else j % len(clouds)]
        tx, ty = 2 * (j % 8), j // 8
        m = np.eye(4, dtype=f32)
        m[:3, 3] = _world(16 * tx + 8, 16 * ty + 8)
        listed.append((cloud, lay, B.CloudTransform(m), B.CloudSettings(opacity_adaptive_radius=False)))
    p = B.GaussianSplattingPlugin(0)
    try:
        sc = PK.Scene(p, listed, [0] * 64, MVIEW)
        for device in (False, True):
            out, pick = PK.target(MVIEW, "f32", device), PK.pick_target(MVIEW, device)
            PK.ok(p, sc.call("pick", out, "f32", 0, None, device, pick))
            pk = PK.pick_host(pick, MVIEW)
            rec, ids = p.projected()
            offs = np.cumsum([0] + sc.counts)
            want = set()
            for j, n in enumerate(sc.counts):
                want |= {(j, 0), (j, n - 1)}
            ent = np.searchsorted(offs, ids, side="right") - 1
            got_vis = {(int(e), int(g - offs[e])) for e, g in zip(ent, ids)}
            assert got_vis == want   # exactly the first and last gaussian of every entity are drawn
            seen = set()
            for r, (e, g) in enumerate(zip(ent, ids)):
                px, py = int(np.floor(rec[r, 0])), int(np.floor(rec[r, 1]))
                j, i = int(e), int(g - offs[e])
                tx, ty = 2 * (j % 8) + (1 if i == sc.counts[j] - 1 and sc.counts[j] > 1 else 0), j // 8
                assert (px // 16, py // 16) == (tx, ty), (j, i, px, py)   # alone on its own tile
                assert (int(pk["entity"][py, px]), int(pk["index"][py, px])) == (j, i), (j, i)
                seen.add((j, i))
            assert seen == want
    finally:
        p.destroy()
