"""The last step of every frame -- the blended f32 state of a pixel written into the caller's target (csrc/raster.cu
write_pixel / store_pixel2 / pack_srgb8 / pack_rgba16f / read_pixel) -- restated in numpy, with the error band of its
approximate sRGB transfer functions, ramp targets that hold every value a channel can take, and one construction per
blend kernel.

Output modes (raster.cu write_pixel), with C the accumulated premultiplied colour and T the remaining transmittance:
  opaque         (C, 1)                                  alpha byte 255 in RGBA8
  premultiplied  (C, 1 - T)
  over           (C + T dst.rgb, (1 - T) + T dst.a)      dst read back from the target in its own format

RGBA8 is sRGB-encoded colour with a linear alpha byte.  The kernel's encoder and decoder use __powf, i.e.
ex2.approx(y * lg2.approx(x)): a byte can differ from the correctly rounded encoding only where 255 enc(c) + 0.5 lies
within `SRGB8_BAND` of an integer.  The band is derived below from the PTX ISA's stated maximum errors, not fitted.
"""
from __future__ import annotations

import dataclasses
import functools

import numpy as np

import bevy_gaussian_splatting_b200 as B
import blend_cases as BC
import kernel_paths as KP

U = 2.0 ** -24                     # unit roundoff of f32
# PTX ISA, lg2.approx.f32: maximum absolute error 2^-22 for inputs in (0.5, 2), maximum relative error 2^-22 for other
# positive finite inputs.  ex2.approx.f32: maximum relative error 2^-22 (2 ulp of a result in [1, 2)).
LG2_ERR = 2.0 ** -22
EX2_ERR = 2.0 ** -22
F32 = np.float32
ENC_LINEAR_MAX = F32(0.0031308)    # raster.cu linear_to_srgb: the linear segment's end, as the f32 constant
DEC_LINEAR_MAX = F32(0.04045)      # raster.cu srgb_decode


# ---------------------------------------------------------------------------------------------------------------------
# float64 formulas (the sRGB transfer functions as specified)

def srgb_encode64(c):
    c = np.clip(np.nan_to_num(np.asarray(c, np.float64), nan=0.0), 0.0, 1.0)
    return np.where(c <= 0.0031308, 12.92 * c, 1.055 * np.power(c, 1 / 2.4) - 0.055)


def srgb_decode64(s):
    s = np.asarray(s, np.float64)
    return np.where(s <= 0.04045, s / 12.92, np.power((s + 0.055) / 1.055, 2.4))


def srgb8_round64(c):
    """The correctly rounded RGBA8 colour byte of a linear value: floor(255 enc(c) + 0.5)."""
    return np.floor(255.0 * srgb_encode64(c) + 0.5)


# ---------------------------------------------------------------------------------------------------------------------
# the kernel's steps in f32 (numpy float32 arithmetic is IEEE round-to-nearest-even, as the kernel's
# mul / add / fma.rn are; __powf is stood in for by the correctly rounded power: its error is the band's business)

def _powf(x, y):
    return np.power(np.asarray(x, np.float64), np.float64(y)).astype(F32)


def linear_to_srgb_f32(c):
    """raster.cu linear_to_srgb: fminf(fmaxf(c, 0), 1) (NaN -> 0), then the two segments in f32."""
    c = np.asarray(c, F32)
    c = np.minimum(np.fmax(c, F32(0)), F32(1)).astype(F32)          # fmaxf(NaN, 0) = 0
    hi = (F32(1.055) * _powf(c, F32(1.0) / F32(2.4)) - F32(0.055)).astype(F32)
    return np.where(c <= ENC_LINEAR_MAX, (F32(12.92) * c).astype(F32), hi).astype(F32)


def byte_of(x):
    """(uint32_t)(x * 255.0f + 0.5f) of an f32 in [0, 1]: two roundings, then truncation."""
    x = np.asarray(x, F32)
    return np.floor(((x * F32(255.0)).astype(F32) + F32(0.5)).astype(F32)).astype(np.uint8)


def pack_srgb8(rgba, with_alpha=True):
    """raster.cu pack_srgb8 of (H, W, 4) f32 -> (H, W, 4) uint8."""
    rgba = np.asarray(rgba, F32)
    out = np.empty(rgba.shape, np.uint8)
    out[..., :3] = byte_of(linear_to_srgb_f32(rgba[..., :3]))
    a = np.minimum(np.fmax(rgba[..., 3], F32(0)), F32(1)).astype(F32)
    out[..., 3] = byte_of(a) if with_alpha else 255
    return out


def pack_rgba16f(rgba):
    """raster.cu pack_rgba16f: __floats2half2_rn, round to nearest even (numpy's f32 -> f16 conversion)."""
    with np.errstate(over="ignore"):
        return np.asarray(rgba, F32).astype(np.float16)


def srgb_decode_f32(byte):
    """raster.cu read_pixel / srgb_decode of a colour byte, f32 steps (the power correctly rounded)."""
    s = (np.asarray(byte, F32) * (F32(1.0) / F32(255.0))).astype(F32)
    lin = (s * (F32(1.0) / F32(12.92))).astype(F32)
    pw = _powf(((s + F32(0.055)).astype(F32) * (F32(1.0) / F32(1.055))).astype(F32), F32(2.4))
    return np.where(s <= DEC_LINEAR_MAX, lin, pw).astype(F32)


def alpha_decode_f32(byte):
    """read_pixel's alpha: (float)(v >> 24) * (1.0f / 255.0f) -- exact in this restatement."""
    return (np.asarray(byte, F32) * (F32(1.0) / F32(255.0))).astype(F32)


def decode_target(dst):
    """The f32 values the kernel reads from a target (RGBA8: rgb up to `srgb_decode_err`; alpha exact)."""
    if dst.dtype == np.uint8:
        return np.concatenate([srgb_decode_f32(dst[..., :3]), alpha_decode_f32(dst[..., 3:])], -1)
    return dst.astype(F32)


def write_pixel(C, T, mode, fmt, dst=None):
    """raster.cu write_pixel for whole frames: C (H, W, 3) f32, T (H, W) f32 -> the target's bytes (as its dtype)."""
    C, T = np.asarray(C, F32), np.asarray(T, F32)[..., None]
    if mode == "over":
        d = decode_target(dst)
        rgb = (T.astype(np.float64) * d[..., :3] + C).astype(F32)        # fmaf: one rounding
        a = (T.astype(np.float64) * d[..., 3:] + (F32(1) - T)).astype(F32)
    else:
        rgb = C
        a = (F32(1) - T).astype(F32) if mode == "premultiplied" else np.ones_like(T)
    out = np.concatenate([rgb, a], -1).astype(F32)
    if fmt == "rgba32f":
        return out
    if fmt == "rgba16f":
        return pack_rgba16f(out)
    return pack_srgb8(out, with_alpha=mode != "opaque")


# ---------------------------------------------------------------------------------------------------------------------
# the RGBA8 error band

def _pow_rel_err(x, y):
    """Relative error bound of __powf(x, y) = ex2.approx(fl(y_f32 * lg2.approx(x))) against x^y exactly, x in (0, 1]:
    lg2.approx's error (absolute 2^-22 on (0.5, 2), relative 2^-22 below), y's f32 rounding and the product's
    rounding (2 U |z|) move the exponent z = y lg2 x; 2^z then moves by ln 2 dz relative; ex2.approx adds 2^-22."""
    L = np.abs(np.log2(x))
    dL = LG2_ERR * np.maximum(1.0, L)
    dz = abs(y) * dL * (1 + 2 * U) + 2.0 * U * abs(y) * L
    return np.expm1(np.log(2.0) * dz) + EX2_ERR * (1 + np.log(2.0) * dz)


def srgb8_encode_err(c):
    """Bound on |255 enc_kernel(c) + 0.5 - (255 enc(c) + 0.5)| for f32 c in [0, 1] (kernel: all its f32 roundings and
    __powf; formula: float64 with exact constants).  Power segment: __powf's relative error on p = c^(1/2.4), the
    rounding of 1.055f (U) and of the product (U), of 0.055f (U 0.055) and the subtraction (U enc), then x 255 (U) and
    + 0.5 (U 256).  Near the segments' joint the f32 and exact thresholds may pick different segments: their values there
    differ by < 1e-7, inside the same bound."""
    c = np.clip(np.asarray(c, np.float64), 0.0, 1.0)
    p = np.power(np.maximum(c, 1e-30), 1 / 2.4)
    e = srgb_encode64(c)
    pw = 1.055 * p * (_pow_rel_err(np.maximum(c, 1e-30), 1 / 2.4) + 3 * U) + 0.055 * U + e * U + 1e-7
    lin = 12.92 * c * 3 * U
    err_enc = np.where(c <= 0.0031308 * (1 + 4 * U), np.maximum(lin, 1e-7 * (c > 0.0031308 * (1 - 4 * U))), pw)
    return 255.0 * (err_enc + e * U) + 256.0 * U


def _max_encode_err():
    c = np.concatenate([np.linspace(0.0, 1.0, 200001), np.geomspace(1e-6, 1.0, 20001)])
    return float(srgb8_encode_err(c).max())


SRGB8_BAND = _max_encode_err()     # ~1.3e-4 of a byte step


def srgb_decode_err(byte):
    """Bound on |srgb_decode_kernel(byte) - srgb_decode64(byte / 255)|: the f32 roundings of byte * (1/255.f) (2 U),
    + 0.055f and * (1/1.055f) (3 U relative on the base, times the exponent 2.4), then __powf; linear segment 3 U."""
    s = np.asarray(byte, np.float64) / 255.0
    d = srgb_decode64(s)
    base = (s + 0.055) / 1.055
    pw = d * (_pow_rel_err(np.maximum(base, 1e-30), 2.4) * (1 + 1e-6) + 2.4 * 5 * U + U)
    return np.where(s <= 0.04045, d * 3 * U, pw) + 1e-12


def in_band(c, extra=0.0):
    """Channels whose RGBA8 byte may differ from `srgb8_round64(c)`: 255 enc(c) + 0.5 within the band (+ `extra`, per
    channel, in byte units) of an integer."""
    x = 255.0 * srgb_encode64(c) + 0.5
    return np.abs(x - np.round(x)) <= SRGB8_BAND + extra


def srgb_encode_slope(c):
    """d(255 enc) / dc, the largest over [c, 1] (enc is concave), capped by the linear segment's 255 * 12.92."""
    c = np.clip(np.asarray(c, np.float64), 0.0, 1.0)
    s = np.where(c <= 0.0031308, 12.92, 1.055 / 2.4 * np.power(np.maximum(c, 0.0031308), 1 / 2.4 - 1.0))
    return 255.0 * np.minimum(s, 12.92)


# ---------------------------------------------------------------------------------------------------------------------
# ramp targets: every value a channel can hold

def ramp_target(fmt: str, h: int, w: int, seed: int = 3) -> np.ndarray:
    """RGBA8: every byte value in every channel.  RGBA16F: every 16-bit pattern in every channel (+-0, subnormals,
    +-inf, NaNs).  RGBA32F: those half values widened, plus f32 specials (+-0, the smallest and largest subnormals,
    +-inf, quiet and signalling NaN payloads) and random bit patterns.  Channels use different strides, so that one
    pixel's four channels are unrelated."""
    n = h * w
    i = np.arange(n, dtype=np.int64)
    strides, offs = (1, 257, 4099, 30001), (0, 11, 101, 997)
    if fmt == "rgba8_srgb":
        assert n >= 256
        return np.stack([((i * s + o) % 256) for s, o in zip(strides, offs)], -1).astype(np.uint8).reshape(h, w, 4)
    assert n >= 65536, "a ramp of every half needs >= 65536 pixels"
    bits16 = np.stack([((i * s + o) % 65536) for s, o in zip(strides, offs)], -1).astype(np.uint16).reshape(h, w, 4)
    if fmt == "rgba16f":
        return bits16.view(np.float16)
    out = bits16.view(np.float16).astype(np.float32)
    rng = np.random.default_rng(seed)
    flat = out.reshape(-1).view(np.uint32)
    specials = np.array([0x00000000, 0x80000000, 0x00000001, 0x007FFFFF, 0x80000001, 0x807FFFFF, 0x7F800000, 0xFF800000,
                         0x7FC00000, 0xFFC00001, 0x7F800001, 0x7FA5A5A5, 0x00800000, 0x7F7FFFFF], np.uint32)
    pick = rng.choice(flat.size, flat.size // 4, replace=False)
    flat[pick] = rng.integers(0, 2 ** 32, pick.size, dtype=np.uint64).astype(np.uint32)
    flat[pick[: specials.size * 64]] = np.tile(specials, 64)
    return out


def seeded_target(fmt: str, h: int, w: int, seed: int) -> np.ndarray:
    """A premultiplied target of ordinary values (alpha in [0, 1], colour <= alpha) in the format."""
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.0, 1.0, (h, w, 4)).astype(np.float32)
    d[..., :3] *= d[..., 3:4]
    if fmt == "rgba16f":
        return d.astype(np.float16)
    if fmt == "rgba8_srgb":
        return np.concatenate([srgb8_round64(d[..., :3]), np.floor(d[..., 3:] * 255 + 0.5)], -1).astype(np.uint8)
    return d


def same_bytes(a, b, allow_negzero=True):
    """Byte-identical, except -0 -> +0 in the float formats (fmaf(1, -0, +0) = +0) and NaN -> any NaN."""
    if a.dtype == np.uint8:
        return a == b
    ia, ib = a.view(np.uint16 if a.dtype == np.float16 else np.uint32), b.view(np.uint16 if b.dtype == np.float16 else np.uint32)
    ok = ia == ib
    if allow_negzero:
        ok |= (a == 0) & (b == 0) & ~np.signbit(a)
    ok |= np.isnan(a) & np.isnan(b)
    return ok


# ---------------------------------------------------------------------------------------------------------------------
# constructions: one frame per blend kernel

W, H = 331, 207                    # odd * odd pixels (odd RGBA8 slot offsets), partial edge tiles, >= 65536 pixels
PATHS = ("r0", "r0aux", "aabb3d", "aabb3d-aux", "aabb2d", "aabb2d-aux", "r2", "rounds")
KERNEL = {"r0": "raster_kernel<0, false, false, false, OneView>", "r0aux": "raster_kernel<0, true, false, false, OneView>",
          "aabb3d": "raster_kernel<1, false, false, false, OneView>", "aabb3d-aux": "raster_kernel<1, true, false, false, OneView>",
          "aabb2d": "raster_kernel<2, false, false, false, OneView>", "aabb2d-aux": "raster_kernel<2, true, false, false, OneView>",
          "r2": "raster2_kernel<false>", "rounds": "raster2_kernel<true>"}
GEOM = {"r0": "obb3d", "r0aux": "obb3d", "aabb3d": "aabb3d", "aabb3d-aux": "aabb3d", "aabb2d": "aabb2d",
        "aabb2d-aux": "aabb2d", "r2": "obb3d", "rounds": "obb3d"}


@dataclasses.dataclass
class Case:
    path: str
    cloud: B.PlanarGaussian3d
    view: object
    settings: B.CloudSettings

    @property
    def aux(self) -> bool:
        return self.path.endswith("aux")

    @property
    def aabb(self) -> bool:
        return BC.GEOMETRIES[GEOM[self.path]][1]

    @property
    def hinted(self) -> bool:
        """raster2_kernel<false> is chosen from the previous frame's counts: render once before the frame under test."""
        return self.path == "r2"


def splat_cloud(view, n: int, half_px, seed: int, dist=(3.0, 30.0), opacity=(0.05, 1.0), margin: float = 0.25):
    """n translucent splats over the middle of the frame (a margin of empty tiles all round), colours over [0, 1]."""
    rng = np.random.default_rng(seed)
    w, h = view.width, view.height
    sp = BC.Splats(view)
    cx = rng.uniform(margin * w, (1 - margin) * w, n)
    cy = rng.uniform(margin * h, (1 - margin) * h, n)
    d = np.sort(rng.uniform(*dist, n))
    _, _, t = sp.depth(cx, cy, d)
    r = rng.uniform(*half_px, n)
    aniso = rng.uniform(1.0, 2.5, n)
    theta = rng.uniform(-np.pi, np.pi, n)
    op = rng.uniform(*opacity, n)
    c = np.array([BC.cutoff_of(B.CloudSettings(), o) for o in op])
    rgb = rng.uniform(0.0, 1.0, (n, 3)).astype(np.float32)
    rgb[: n // 8] = rng.choice([0.0, 1.0], (n // 8, 3))                 # exact 0 / 1 colours too
    return sp.cloud(cx, cy, d, sp.scale_for(r, t, c), sp.scale_for(r / aniso, t, c), theta, op, rgb)


@functools.lru_cache(maxsize=None)
def case(path: str) -> Case:
    view = B.headless_view(W, H)
    geom = GEOM[path]
    s = BC.settings_for(geom, saturated=False, binning_rounds=(path == "rounds"))
    if path == "r2":
        cloud = splat_cloud(view, 120, (24.0, 60.0), seed=21)          # >= 8 (splat, tile) pairs per visible splat
    else:
        cloud = splat_cloud(view, 400, (1.5, 12.0), seed=11 + PATHS.index(path))
    return Case(path, cloud, view, s)


def frame_counts(oracle, c: Case):
    u = B.GaussianSplattingPlugin.cloud_uniform(c.settings)
    til = oracle.render_tiles(c.cloud, c.view.to_abi(), u, c.settings.to_abi(), want_image=False)
    return til["n_vis"], til["n_pairs"]


def reaches(oracle, c: Case) -> bool:
    """The frame under test takes the case's kernel (api.cu plan_frame, raster.cu launch_raster), from the oracle's
    counts, which the library's binning reproduces exactly."""
    n_vis, n_pairs = frame_counts(oracle, c)
    tiles = KP.num_tiles(c.view.width, c.view.height)
    mode = 0 if not c.aabb else (1 if c.settings.gaussian_mode == B.GaussianMode.Gaussian3d else 2)
    rounds = KP.chunked(tiles, mode, c.aux, c.settings.binning_rounds, n_vis, n_pairs)
    large = KP.large_footprint_raster(n_vis, n_pairs) if c.hinted else False
    # what the frame under test (the second one when hinted) runs
    if c.path == "rounds":
        return rounds and mode == 0 and not c.aux
    if c.path == "r2":
        return mode == 0 and large and not rounds
    # raster_kernel<mode, aux>: never rounds; for mode 0 the next frame (the other formats) must not turn large either
    return not rounds and (mode != 0 or not KP.large_footprint_raster(n_vis, n_pairs)) and mode == {"obb3d": 0, "aabb3d": 1, "aabb2d": 2}[GEOM[c.path]]


# the frame whose pair list overflows a fresh context's buffer (api.cu render_impl: max(n, 2^20) pairs)
REGROW_W, REGROW_H = 1280, 720


@functools.lru_cache(maxsize=None)
def regrow_case(rounds: bool) -> Case:
    view = B.headless_view(REGROW_W, REGROW_H)
    s = BC.settings_for("obb3d", saturated=False, binning_rounds=rounds)
    # big, faint splats: > 2^20 pairs, and no tile saturates (a chunked frame would skip its later rounds)
    cloud = splat_cloud(view, 7000, (90.0, 160.0), seed=5, opacity=(0.004, 0.02), margin=0.0)
    return Case("rounds" if rounds else "r0", cloud, view, s)


def chain_clouds(view, k: int = 4):
    """k clouds, far to near: cloud j lies at distances [24 - 5 j, 28 - 5 j)."""
    return [splat_cloud(view, 300, (2.0, 16.0), seed=40 + j, dist=(24.0 - 5 * j, 28.0 - 5 * j)) for j in range(k)]
