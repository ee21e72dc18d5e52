"""Every blend kernel's coverage decisions bit for bit, and its pixel values against per-pixel error bounds.

Each variant of csrc/raster.cu is reached through the selection rules restated in `kernel_paths`:
  r0      raster_kernel<0, false>   USE_OBB first frame of a fresh context (no hints: not large_footprint_raster)
  r0aux   raster_kernel<0, true>    the same frame through render_view_aux
  r2      raster2_kernel<false>     the hinted second frame of a heavy frame, once large_footprint_raster holds
  rounds  raster2_kernel<true>      binning_rounds=True, the knife pairs in a round after the first
  aabb3d  raster_kernel<1, *>       3DGS USE_AABB (colour, and aux)
  aabb2d  raster_kernel<2, *>       2DGS USE_AABB (colour, and aux)
  obb2d   raster_kernel<0, false>   2DGS USE_OBB surfel records (uy = vx = 0)
and rendered in three output modes: over an opaque clear, premultiplied (C, 1 - T), and blended over a seeded RGBA32F
target (C + T dst.rgb, (1 - T) + T dst.a).

* Saturated frames (tests/blend_cases.py): every pixel whose blended alphas are all the clamp must be within 4 ulps of
  the channel magnitude of the oracle's f32 frame.  A flipped coverage decision of its first or second covering splat
  moves such a pixel by >= 1e-4, so this holds the frame to the oracle's coverage map; a failure names the pixel, its
  first splat and the pair class when it is a knife pair.
* Every frame: |frame - expected| <= bound per pixel and channel, where expected is composed from the trace's float64
  blend and the bound is `blend_cases.frame_bounds` (derived in `blend_bounds`: the alpha error of ex2.approx / __expf
  and the rounding of their argument propagated through T, f32 accumulation rounding, the colour records' difference
  from the oracle's, and T_STOP m where the stop may fall one splat apart).
* RGBA16F and RGBA8-sRGB frames are the f16 rounding / 8-bit sRGB encoding of some value inside each pixel's error
  interval.
"""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import blend_cases as BC
import kernel_paths as KP

pytestmark = pytest.mark.gpu

OUT_MODES = ("opaque", "premultiplied", "over")
REPORT = {}


def uniform(s, h=None):
    return B.GaussianSplattingPlugin.cloud_uniform(s, None, h.aabb if h is not None else None)


def render(p, h, s, view, out_mode, fmt="rgba32f", dst=None):
    """One frame into a device target (torch), which for `over` holds `dst` first."""
    import torch

    code, dtype, _ = B.GaussianSplattingPlugin.FORMATS[fmt]
    tdt = {np.float32: torch.float32, np.float16: torch.float16, np.uint8: torch.uint8}[dtype]
    tgt = torch.zeros((view.height, view.width, 4), dtype=tdt, device="cuda")
    if dst is not None:
        tgt.copy_(torch.from_numpy(np.ascontiguousarray(dst)))
    torch.cuda.synchronize()
    u, st = p._uniform_and_settings(h, s, None, False, out_mode == "premultiplied", out_mode == "over")
    v = view.to_abi()
    p._check(p._lib.bgs_render(p._ctx, h._h, C.byref(v), C.byref(u), C.byref(st), C.c_void_p(tgt.data_ptr()), code, 1))
    torch.cuda.synchronize()
    return tgt.cpu().numpy()


def seeded_target(view, seed, fmt="rgba32f"):
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.0, 1.0, (view.height, view.width, 4)).astype(np.float32)
    d[..., :3] *= d[..., 3:4]                       # premultiplied
    if fmt == "rgba16f":
        return d.astype(np.float16)
    if fmt == "rgba8_srgb":
        c = np.clip(d[..., :3], 0, 1)
        enc = np.where(c <= 0.0031308, 12.92 * c, 1.055 * np.power(c, 1 / 2.4) - 0.055)
        return np.concatenate([np.floor(enc * 255 + 0.5), np.floor(d[..., 3:4] * 255 + 0.5)], -1).astype(np.uint8)
    return d


def check_records(p, oracle, cloud, s, view, h):
    """Projected records bit-exact (as check_against_oracle); -> (trace, max |colour_gpu - colour_oracle|)."""
    u = uniform(s, h)
    til = oracle.render_tiles(cloud, view.to_abi(), u, s.to_abi(), want_image=False)
    rec, ids = p.projected()
    assert np.array_equal(ids, til["rank_to_id"])
    orec = oracle.project(cloud, view.to_abi(), u, s.to_abi(), ids)
    drawn = orec["xlo"] <= orec["xhi"]
    if s.aabb and s.gaussian_mode == B.GaussianMode.Gaussian3d:
        geo = np.stack([orec["cx"], orec["cy"], orec["extra"][:, 0], orec["extra"][:, 1], orec["extra"][:, 2], orec["extra"][:, 3]], 1)
    else:
        geo = np.stack([orec[k] for k in ("cx", "cy", "ux", "uy", "vx", "vy")], 1)
    assert np.array_equal(rec[drawn, :6].view(np.uint32), geo[drawn].view(np.uint32)), "projected geometry not bit-exact"
    col = np.stack([orec[k] for k in ("r", "g", "b")], 1)
    dc = float(np.abs(rec[drawn, 8:11] - col[drawn]).max()) if drawn.any() else 0.0
    assert np.array_equal(rec[drawn, 11].view(np.uint32), orec["op"][drawn].view(np.uint32))
    return til, dc


def assert_within_bound(name, got, trace, aabb, out_mode, dc, dst=None, classes=None, ranks=None):
    want = BC.expected_frame(trace, out_mode, dst)
    bound, _ = BC.frame_bounds(trace, aabb, out_mode, dc, dst)
    err = np.abs(got.astype(np.float64) - want)
    ratio = np.where(err > 0, err / np.maximum(bound, 1e-300), 0.0)
    worst = np.unravel_index(int(ratio.argmax()), ratio.shape)
    REPORT[name] = max(REPORT.get(name, 0.0), float(ratio.max()))
    assert ratio.max() <= 1.0, (f"{name}: pixel (x={worst[1]}, y={worst[0]}) channel {worst[2]} err {err[worst]:.3g} > bound "
                                f"{bound[worst]:.3g}; first splat rank {trace['rank0'][worst[:2]]}, {pair_name(worst, classes, ranks)}")
    return float(ratio.max())


def pair_name(yx, classes, ranks):
    if classes is None:
        return "not a knife pixel"
    y, x = yx[0], yx[1]
    names = [k for k, v in classes[0].items() for i in v if tuple(classes[1][i]) == (x, y)]
    return f"knife pair classes {names}" if names else "not a knife pixel"


def ulps4(got, want):
    """|got - want| <= 4 ulp of the channel magnitude (f32)."""
    mag = np.maximum(np.abs(want), np.float32(2.0 ** -20)).astype(np.float32)
    return np.abs(got.astype(np.float64) - want.astype(np.float64)) <= 4 * np.spacing(mag).astype(np.float64)


def assert_coverage_map(name, got, oracle_img, trace, out_mode, classes=None):
    """Saturated frame: pixels whose blended alphas are all the clamp match the oracle's f32 frame to 4 ulps."""
    exact = (trace["flags"] & 4) == 0
    want = oracle_img.copy()
    if out_mode == "premultiplied":
        want[..., 3] = np.float32(1) - trace["T"]
    ok = ulps4(got, want) if out_mode != "over" else np.ones_like(got, bool)
    bad = np.argwhere(~ok.all(-1) & exact)
    if len(bad):
        y, x = bad[0]
        raise AssertionError(f"{name}: {len(bad)} saturated pixels off the oracle's coverage map, first (x={x}, y={y}): "
                             f"got {got[y, x]} want {want[y, x]}; blended ranks {trace['rank0'][y, x]}, {trace['rank1'][y, x]}; "
                             f"{pair_name((y, x), classes, None)}")


def assert_quantised(got, trace, aabb, out_mode, fmt, dc, dst=None):
    """RGBA16F / RGBA8-sRGB: the format's rounding of some value inside each pixel's interval [want - b, want + b]."""
    want = BC.expected_frame(trace, out_mode, dst)
    b, _ = BC.frame_bounds(trace, aabb, out_mode, dc, dst)
    lo, hi = want - b, want + b
    if fmt == "rgba16f":
        def q(x):
            return np.float16(x).astype(np.float64) if np.isscalar(x) else x.astype(np.float16).astype(np.float64)
        g = got.astype(np.float64)
        ok = (g >= q(lo)) & (g <= q(hi))
    else:
        def enc(c):
            c = np.clip(c, 0, 1)
            return np.where(c <= 0.0031308, 12.92 * c, 1.055 * np.power(c, 1 / 2.4) - 0.055)
        eps = 1e-5                                    # __powf in the kernel's encoder
        g = got.astype(np.float64)
        lo8 = np.floor(np.concatenate([enc(lo[..., :3]) - eps, np.clip(lo[..., 3:], 0, 1)], -1) * 255 + 0.5)
        hi8 = np.floor(np.concatenate([enc(hi[..., :3]) + eps, np.clip(hi[..., 3:], 0, 1)], -1) * 255 + 0.5)
        if out_mode == "opaque":
            lo8[..., 3] = hi8[..., 3] = 255
        ok = (g >= lo8) & (g <= hi8)
    bad = np.argwhere(~ok)
    assert len(bad) == 0, f"{fmt} {out_mode}: {len(bad)} channels outside the rounding of their interval, first {bad[0]}"


# ---------------------------------------------------------------------------------------------------------------------

VARIANTS = ["r0", "r0aux", "r2", "rounds", "aabb3d", "aabb2d", "obb2d", "aabb3d-aux", "aabb2d-aux"]
GEOM = {"r0": "obb3d", "r0aux": "obb3d", "r2": "obb3d", "rounds": "obb3d", "aabb3d": "aabb3d", "aabb2d": "aabb2d",
        "obb2d": "obb2d", "aabb3d-aux": "aabb3d", "aabb2d-aux": "aabb2d"}


def frames(oracle, variant):
    """(label, cloud, view, settings, knife classes or None, saturated) of a variant."""
    geom = GEOM[variant]
    out = []
    if variant != "r2":
        cloud, view, s = BC.saturated_case(geom)
        if variant == "rounds":
            s = dataclasses.replace(s, binning_rounds=True)
        out.append(("saturated", cloud, view, s, None, True))
    for sat in (True, False):
        case = BC.knife_case(oracle, geom, sat, heavy=(variant == "r2"))
        s = case.settings
        if variant == "rounds":
            s = dataclasses.replace(s, binning_rounds=True)
        cls, _ = BC.pair_classes(oracle, case)
        out.append(("knife-sat" if sat else "knife", case.cloud, case.view, s, (cls, case.pixels), sat))
    return out


def run_path(p, h, s, view, variant, out_mode, fmt="rgba32f", dst=None):
    """Render through the variant's kernel and assert the path was taken."""
    if variant.endswith("aux") or variant == "r0aux":
        assert out_mode == "opaque"
        colour, _, _ = p.render_view_aux(h, s, view, fmt=fmt)
        return colour
    if variant == "r2":
        p.render_view(h, s, view, fmt=fmt)          # sets the hints
        fs = p.frame_stats()
        assert KP.large_footprint_raster(fs.n_visible, fs.n_pairs), (fs.n_visible, fs.n_pairs)
        assert not KP.chunked(fs.tiles_x * fs.tiles_y, flag=False)
    img = render(p, h, s, view, out_mode, fmt, dst)
    fs = p.frame_stats()
    if variant == "rounds":
        assert fs.rounds > 1
    else:
        assert fs.rounds == 1
    if variant in ("r0", "obb2d"):   # the next frame (quantised formats) stays on raster_kernel<0> too
        assert not KP.large_footprint_raster(fs.n_visible, fs.n_pairs)
    return img


@pytest.mark.parametrize("variant", VARIANTS)
def test_blend_variant_vs_oracle(oracle, variant):
    geom = GEOM[variant]
    aabb = BC.GEOMETRIES[geom][1]
    modes = ("opaque",) if variant.endswith("aux") else OUT_MODES
    for label, cloud, view, s, classes, sat in frames(oracle, variant):
        name = f"{variant}/{label}"
        u = uniform(s)
        trace = oracle.blend_trace(cloud, view.to_abi(), u, s.to_abi())
        oimg = oracle.render_tiles(cloud, view.to_abi(), u, s.to_abi())["image"]
        if classes is not None:
            if variant == "rounds":
                assert len(classes[0]["ROUND_GE1"]) > 0        # knife pairs in a round after the first
            print(f"\n{name} knife pairs: " + ", ".join(f"{k} {len(v)}" for k, v in classes[0].items() if v))
        # the projected records, bit-exact geometry, and dc = max |colour_gpu - colour_oracle| of the drawn records: the
        # records are the same whatever the output mode or raster kernel, so one plain frame measures dc for all of them
        p = B.GaussianSplattingPlugin(0)
        try:
            h = p.add_cloud(cloud)
            p.render_view(h, dataclasses.replace(s, binning_rounds=False), view)
            _, dc = check_records(p, oracle, cloud, s, view, h)
            h.destroy()
        finally:
            p.destroy()
        for out_mode in modes:
            p = B.GaussianSplattingPlugin(0)          # a fresh context per frame: no hints from another one
            try:
                h = p.add_cloud(cloud)
                dst = seeded_target(view, 7) if out_mode == "over" else None
                got = run_path(p, h, s, view, variant, out_mode, dst=dst)
                if sat:
                    assert_coverage_map(name + "/" + out_mode, got, oimg, trace, out_mode, classes)
                assert_within_bound(name, got, trace, aabb, out_mode, dc, dst, classes)
                if out_mode != "over" and not variant.endswith("aux") and variant != "r0aux":
                    for fmt in ("rgba16f", "rgba8_srgb"):
                        q = run_path(p, h, s, view, variant, out_mode, fmt)
                        assert_quantised(q, trace, aabb, out_mode, fmt, dc)
                h.destroy()
            finally:
                p.destroy()
    print(f"\nerr/bound {variant}: " + ", ".join(f"{k} {v:.3f}" for k, v in REPORT.items() if k.startswith(variant + "/")))
