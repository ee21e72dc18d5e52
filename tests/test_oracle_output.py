"""CPU checks of tests/output_cases.py: the f32 restatement of the frame's output step against the float64 formulas
outside the derived RGBA8 band, the ramp targets' coverage of every channel value, and each construction reaching the
blend kernel it exists for."""
import numpy as np
import pytest

import kernel_paths as KP
import output_cases as OC


def _f32_sweep():
    """Every f32 in [0, 1] would be 2^30 values: a dense sweep, the ties' neighbourhoods and the segment joint."""
    c = np.linspace(0.0, 1.0, 400001, dtype=np.float64).astype(np.float32)
    ties = OC.srgb_decode64((np.arange(256) + 0.5) / 255.0)       # 255 enc(c) + 0.5 is an integer there
    near = (ties.astype(np.float32)[:, None].view(np.int32) + np.arange(-64, 65, dtype=np.int32)[None, :]).view(np.float32)
    joint = (np.float32(0.0031308).view(np.int32) + np.arange(-256, 257, dtype=np.int32)).view(np.float32)
    return np.unique(np.concatenate([c, near.reshape(-1), joint, np.float32([0.0, 1.0, -0.0, 2.0, -1.0])]))


def test_band_is_derived_small():
    """The band comes from the PTX error bounds: far below a byte step, above f32 rounding of the byte alone."""
    assert 256 * OC.U < OC.SRGB8_BAND < 1e-3, OC.SRGB8_BAND
    print(f"\nRGBA8 band: +-{OC.SRGB8_BAND:.3g} of a byte step")


def test_restated_encoder_matches_float64_outside_band():
    c = _f32_sweep()
    got = OC.byte_of(OC.linear_to_srgb_f32(c)).astype(np.float64)
    want = OC.srgb8_round64(c)
    band = OC.in_band(c)
    assert np.array_equal(got[~band], want[~band]), c[~band][got[~band] != want[~band]][:8]
    assert np.all(np.abs(got - want) <= 1)
    # the sweep reaches the band (the ties' neighbourhoods), so the exclusion is not vacuous; on a uniform sweep the band
    # holds about 2 x band of the channels
    assert band.sum() > 0
    u = np.linspace(0.0, 1.0, 400001, dtype=np.float64).astype(np.float32)
    assert OC.in_band(u).mean() < 10 * OC.SRGB8_BAND


def test_restated_alpha_and_half_rounding():
    a = np.linspace(0.0, 1.0, 100001, dtype=np.float32)
    got = OC.byte_of(a).astype(np.float64)
    # (x * 255.0f + 0.5f): f32 product and sum; never more than the one rounding away from floor(255 a + 0.5)
    assert np.all(np.abs(got - np.floor(255.0 * a.astype(np.float64) + 0.5)) <= 1)
    for k in range(256):                                       # a decoded alpha byte encodes back to itself
        assert OC.byte_of(OC.alpha_decode_f32(np.uint8(k))) == k
    h = OC.pack_rgba16f(np.float32([1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 65520.0, -0.0, 6e-8]))
    assert h.view(np.uint16).tolist() == [0x3C00, 0x3C02, 0x7C00, 0x8000, 0x0001]   # ties to even, overflow to inf


def test_decode_encode_round_trip_is_identity():
    """An RGBA8 pixel no splat blends is decoded and encoded again by raster2_kernel in blend-over mode: identity for all
    256 colour bytes even at the decoder's and encoder's error bounds."""
    k = np.arange(256)
    d = OC.srgb_decode64(k / 255.0)
    x = 255.0 * OC.srgb_encode64(d) + 0.5
    slack = OC.SRGB8_BAND + OC.srgb_encode_slope(np.maximum(d - OC.srgb_decode_err(k), 0)) * OC.srgb_decode_err(k)
    assert np.array_equal(np.floor(x), k) and np.all(np.abs(x - np.round(x)) > slack)
    assert np.array_equal(OC.byte_of(OC.linear_to_srgb_f32(OC.srgb_decode_f32(k))), k)


def test_write_pixel_restatement_modes():
    rng = np.random.default_rng(0)
    C = rng.uniform(0, 1, (8, 9, 3)).astype(np.float32)
    T = rng.uniform(0, 1, (8, 9)).astype(np.float32)
    dst = OC.seeded_target("rgba32f", 8, 9, 1)
    op = OC.write_pixel(C, T, "opaque", "rgba32f")
    assert np.array_equal(op[..., :3], C) and np.all(op[..., 3] == 1)
    pm = OC.write_pixel(C, T, "premultiplied", "rgba32f")
    assert np.array_equal(pm[..., 3], np.float32(1) - T)
    ov = OC.write_pixel(C, T, "over", "rgba32f", dst)
    want = C.astype(np.float64) + T[..., None].astype(np.float64) * dst[..., :3]
    assert np.all(np.abs(ov[..., :3] - want) <= 2 * OC.U * np.abs(want) + 1e-30)
    # over a zero target, blend-over and premultiplied agree bit for bit (fmaf(T, 0, C) = C, fmaf(T, 0, 1 - T) = 1 - T)
    assert np.array_equal(OC.write_pixel(C, T, "over", "rgba32f", np.zeros_like(dst)), pm)
    assert OC.write_pixel(C, T, "opaque", "rgba8_srgb")[..., 3].min() == 255


@pytest.mark.parametrize("fmt", ["rgba8_srgb", "rgba16f", "rgba32f"])
def test_ramp_targets_hold_every_value(fmt):
    r = OC.ramp_target(fmt, OC.H, OC.W)
    if fmt == "rgba8_srgb":
        for ch in range(4):
            assert np.unique(r[..., ch]).size == 256
    elif fmt == "rgba16f":
        for ch in range(4):
            assert np.unique(r[..., ch].view(np.uint16)).size == 65536
        assert np.isnan(r).any() and np.isposinf(r).any() and np.isneginf(r).any()
        assert (r.view(np.uint16) == 0x8000).any() and ((r.view(np.uint16) & 0x7C00) == 0).sum() > 1000   # -0, subnormals
    else:
        b = r.view(np.uint32)
        for bits in (0x80000000, 0x00000001, 0x807FFFFF, 0x7F800000, 0xFF800000, 0x7FA5A5A5, 0xFFC00001):
            assert (b == bits).any(), hex(bits)
        assert np.isnan(r).sum() > 100 and ((b & 0x7F800000) == 0).sum() > 100


@pytest.mark.parametrize("path", OC.PATHS)
def test_construction_reaches_its_kernel(oracle, path):
    c = OC.case(path)
    assert OC.reaches(oracle, c), (path, OC.frame_counts(oracle, c))
    n_vis, n_pairs = OC.frame_counts(oracle, c)
    u = OC.B.GaussianSplattingPlugin.cloud_uniform(c.settings)
    trace = oracle.blend_trace(c.cloud, c.view.to_abi(), u, c.settings.to_abi())
    untouched = trace["n_blended"] == 0
    # pixels no splat blends: whole empty tiles and uncovered pixels of non-empty ones
    til = oracle.render_tiles(c.cloud, c.view.to_abi(), u, c.settings.to_abi(), want_image=False)
    empty = (til["tile_ranges"][:, 1] == til["tile_ranges"][:, 0]).reshape(-(-c.view.height // 16), -(-c.view.width // 16))
    empty_px = np.repeat(np.repeat(empty, 16, 0), 16, 1)[: c.view.height, : c.view.width]
    assert empty_px.sum() > 1000 and (untouched & ~empty_px).sum() > 100 and (~untouched).sum() > 1000
    print(f"\n{path} ({OC.KERNEL[path]}): n_vis {n_vis} pairs {n_pairs}, untouched {untouched.sum()} "
          f"(in empty tiles {empty_px.sum()})")


@pytest.mark.parametrize("rounds", [False, True])
def test_regrow_construction_overflows_a_fresh_buffer(oracle, rounds):
    c = OC.regrow_case(rounds)
    n_vis, n_pairs = OC.frame_counts(oracle, c)
    cap = KP.initial_pair_capacity(len(c.cloud))
    # a chunked frame's rounds each need their own share; the last round holds 7/8 of the ranks
    assert n_pairs > cap * (1.25 if rounds else 1.0), (n_pairs, cap)
    tiles = KP.num_tiles(c.view.width, c.view.height)
    assert KP.chunked(tiles, flag=c.settings.binning_rounds) == rounds
