"""Host-side cloud container and synthetic generators.

`PlanarGaussian3d` mirrors the reference's struct-of-Vecs (src/gaussian/formats/planar_3d.rs:45-54;
planes in binding order position_visibility, spherical_harmonic, rotation, scale_opacity) as four
C-contiguous float32 numpy arrays -- exactly the four host pointers `bgs_cloud_upload_f32` borrows.

`random_gaussians_3d_seeded` follows the reference generator's distributions and field order
(planar_3d.rs:120-168: rotation 4xU(-1,1) unnormalised; position 3xU(-20,20), visibility 1;
scale 3xU(0,1); opacity U(0,0.8); SH 48xU(-1,1)) with this repo's own counter-based PRNG (numpy
Philox): the reference's ChaCha12 stream is not reproduced bit-for-bit (SURVEY.md §8c).
"""
from __future__ import annotations

import dataclasses

import numpy as np

SH_COEFF_COUNT = 48  # src/material/spherical_harmonics.rs:46-47 (sh3 default)
HALF_SH_COEFF_COUNT = 24
# SH degree d (the reference's sh0 .. sh3 features; include/bgs.h): K_d = (d + 1)^2 coefficients per channel, S_d =
# pad4(3 K_d) floats per gaussian, coefficient k of channel c at sh[3k + c]; lanes 3 K_d .. S_d - 1 are padding
SH_WIDTHS = (4, 12, 28, 48)


def sh_bands(sh_degree: int) -> int:
    """K_d: coefficients per channel at degree d."""
    return (sh_degree + 1) ** 2


def sh_degree_of_width(width: int) -> int:
    """The degree whose SH plane is `width` floats (4, 12, 28 or 48); any other width raises ValueError."""
    if width not in SH_WIDTHS:
        raise ValueError(f"an SH plane holds 4, 12, 28 or 48 floats per gaussian (degree 0..3), not {width}")
    return SH_WIDTHS.index(width)


@dataclasses.dataclass
class PlanarGaussian3d:
    position_visibility: np.ndarray  # (n, 4) f32: x, y, z, visibility      f32.rs:53-56
    spherical_harmonic: np.ndarray   # (n, S_d) f32: sh[3k + c], S_d = 4, 12, 28 or 48 spherical_harmonics.rs:114-120
    rotation: np.ndarray             # (n, 4) f32: w, x, y, z               f32.rs:95-97
    scale_opacity: np.ndarray        # (n, 4) f32: sx, sy, sz, opacity      f32.rs:172-175

    def __post_init__(self):
        sh = np.ascontiguousarray(self.spherical_harmonic, dtype=np.float32)
        if sh.ndim != 2:
            raise ValueError("spherical_harmonic must have shape (n, S_d)")
        sh_degree_of_width(sh.shape[1])
        self.spherical_harmonic = sh
        for name, width in (("position_visibility", 4), ("rotation", 4), ("scale_opacity", 4)):
            a = np.ascontiguousarray(getattr(self, name), dtype=np.float32)
            if a.ndim != 2 or a.shape[1] != width:
                raise ValueError(f"{name} must have shape (n, {width})")
            setattr(self, name, a)
        n = len(self.position_visibility)
        if not (len(self.spherical_harmonic) == len(self.rotation) == len(self.scale_opacity) == n):
            raise ValueError("planes disagree on n")

    def __len__(self) -> int:
        return len(self.position_visibility)

    @property
    def sh_degree(self) -> int:
        """0..3, from the SH plane's width (4, 12, 28, 48)."""
        return sh_degree_of_width(self.spherical_harmonic.shape[1])

    def with_sh_degree(self, sh_degree: int) -> "PlanarGaussian3d":
        """The cloud at another degree: the coefficients of the bands both degrees hold are kept, the others (and every
        padding lane) are zero.  Truncating drops the higher bands; zero-padding to degree 3 gives a cloud that renders
        exactly like this one."""
        if sh_degree not in range(4):
            raise ValueError(f"sh_degree must be 0..3, not {sh_degree}")
        width = SH_WIDTHS[sh_degree]
        keep = 3 * min(sh_bands(sh_degree), sh_bands(self.sh_degree))
        sh = np.zeros((len(self), width), np.float32)
        sh[:, :keep] = self.spherical_harmonic[:, :keep]
        return PlanarGaussian3d(self.position_visibility, sh, self.rotation, self.scale_opacity)

    def subset(self, n) -> "PlanarGaussian3d":
        """An int: the first n gaussians.  An index array: those gaussians, in that order -- what the reference's
        save_selection (src/query/select.rs:156-176) writes out for a selection."""
        if np.ndim(n) == 0:
            return PlanarGaussian3d(self.position_visibility[:n], self.spherical_harmonic[:n], self.rotation[:n],
                                    self.scale_opacity[:n])
        idx = np.asarray(n)
        if idx.dtype.kind not in "iu":
            raise TypeError("subset: indices must be integers")
        return PlanarGaussian3d(self.position_visibility[idx], self.spherical_harmonic[idx], self.rotation[idx],
                                self.scale_opacity[idx])

    # ---- f16 planar layout (src/gaussian/f16.rs:30-56,244-263; planar.wgsl:117-176) -----------------
    def compute_aabb(self) -> tuple[np.ndarray, np.ndarray]:
        """The entity `Aabb` as the render world sees it: `compute_aabb` (src/gaussian/interface.rs:22-66: positions
        +- 0.1) -> `Aabb {center, half_extents}` (src/gaussian/cloud.rs:45-62) -> `aabb.min()` / `aabb.max()`
        (center -+ half_extents, src/render/mod.rs:1070-1071), every step in f32 like glam."""
        return compute_aabb(self.position_visibility)

    @staticmethod
    def from_f16(pos_vis, sh_packed, rot_scale_opacity, sh_degree: int | None = None) -> "PlanarGaussian3d":
        """The exact inverse of `pack_f16`: each half widened to f32 (pack_f16 of the result gives the same words back for
        every non-NaN half; a NaN half stays NaN).  For a precomputed-covariance record the result holds the covariance in
        the slots `precomputed_covariance()` uses.  sh_degree None: the degree of a 2-D sh_packed's width (S_d / 2
        words), 3 for a flat one."""
        def halves(w, shift):
            return ((np.asarray(w, np.uint32) >> np.uint32(shift)) & np.uint32(0xFFFF)).astype(np.uint16).view(np.float16).astype(np.float32)

        shp = np.asarray(sh_packed, np.uint32)
        if sh_degree is None:
            sh_degree = sh_degree_of_width(2 * shp.shape[1]) if shp.ndim == 2 else 3
        if sh_degree not in range(4):
            raise ValueError(f"sh_degree must be 0..3, not {sh_degree}")
        width = SH_WIDTHS[sh_degree]
        shp = shp.reshape(-1, width // 2)
        w = np.asarray(rot_scale_opacity, np.uint32).reshape(-1, 4)
        sh = np.empty((len(shp), width), np.float32)
        sh[:, 0::2], sh[:, 1::2] = halves(shp, 0), halves(shp, 16)     # even coefficient in the low half
        rot = np.stack([halves(w[:, 0], 16), halves(w[:, 0], 0), halves(w[:, 1], 16), halves(w[:, 1], 0)], axis=1)
        so = np.stack([halves(w[:, 2], 16), halves(w[:, 2], 0), halves(w[:, 3], 16), halves(w[:, 3], 0)], axis=1)
        return PlanarGaussian3d(np.asarray(pos_vis, np.float32).reshape(-1, 4), sh, rot, so)

    def pack_f16(self) -> tuple[np.ndarray, np.ndarray]:
        """-> (sh_packed (n, S_d / 2) u32, rot_scale_opacity (n,4) u32); pack(upper, lower) = upper<<16 | lower."""
        def bits(a):
            return np.ascontiguousarray(a, dtype=np.float32).astype(np.float16).view(np.uint16).astype(np.uint32)

        sh = bits(self.spherical_harmonic)
        sh_packed = (sh[:, 1::2] << 16) | sh[:, 0::2]  # even coefficient in the low half
        r, s = bits(self.rotation), bits(self.scale_opacity)
        rso = np.stack([(r[:, 0] << 16) | r[:, 1], (r[:, 2] << 16) | r[:, 3], (s[:, 0] << 16) | s[:, 1],
                        (s[:, 2] << 16) | s[:, 3]], axis=1)
        return np.ascontiguousarray(sh_packed, dtype=np.uint32), np.ascontiguousarray(rso, dtype=np.uint32)

    def precomputed_covariance(self) -> "PlanarGaussian3d":
        """`Covariance3dOpacity` per gaussian (src/gaussian/f32.rs:238-251 <- covariance.rs:4-41, every product in f32, glam's
        accumulation order), laid out in the plane slots `Covariance3dOpacityPacked128` occupies (f16.rs:131-170): rotation
        = (c0, c1, c2, c3), scale_opacity = (c4, c5, opacity, opacity).  `pack_f16()` of the result is the record the
        reference's PRECOMPUTE_COVARIANCE_3D layout uploads; `rounded_to_f16()` is what its shader decodes."""
        f = np.float32
        q, so = self.rotation.astype(f), self.scale_opacity.astype(f)
        r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
        two, one = f(2.0), f(1.0)
        R = np.empty((len(q), 3, 3), f)     # R[:, i, j]: row i, column j (columns = the triplets covariance.rs writes)
        R[:, 0, 0] = one - two * (y * y + z * z); R[:, 1, 0] = two * (x * y - r * z); R[:, 2, 0] = two * (x * z + r * y)
        R[:, 0, 1] = two * (x * y + r * z); R[:, 1, 1] = one - two * (x * x + z * z); R[:, 2, 1] = two * (y * z - r * x)
        R[:, 0, 2] = two * (x * z - r * y); R[:, 1, 2] = two * (y * z + r * x); R[:, 2, 2] = one - two * (x * x + y * y)
        M = (so[:, :3, None] * R).astype(f)                      # M = S R: row i scaled by s_i
        def sg(i, j):
            return ((M[:, 0, i] * M[:, 0, j] + M[:, 1, i] * M[:, 1, j]).astype(f) + M[:, 2, i] * M[:, 2, j]).astype(f)
        cov_rot = np.stack([sg(0, 0), sg(0, 1), sg(0, 2), sg(1, 1)], axis=1)
        cov_so = np.stack([sg(1, 2), sg(2, 2), so[:, 3], so[:, 3]], axis=1)
        return PlanarGaussian3d(self.position_visibility, self.spherical_harmonic, cov_rot, cov_so)

    def rounded_to_f16(self) -> "PlanarGaussian3d":
        """The f32 cloud the f16 layout decodes to (position stays f32: bindings.wgsl:104-106)."""
        def rt(a):
            return a.astype(np.float16).astype(np.float32)

        return PlanarGaussian3d(self.position_visibility, rt(self.spherical_harmonic), rt(self.rotation),
                                rt(self.scale_opacity))


def compute_aabb(position_visibility: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """`PlanarGaussian3d.compute_aabb` of an (n, 4) position plane."""
    p = np.asarray(position_visibility, np.float32)[:, :3]
    if not len(p):
        return aabb_of_extent(np.full(3, np.inf, np.float32), np.full(3, -np.inf, np.float32))
    return aabb_of_extent(p.min(0), p.max(0))


def aabb_of_extent(pmin, pmax) -> tuple[np.ndarray, np.ndarray]:
    """`compute_aabb`'s steps from the per-axis min and max of the positions (+inf / -inf for none): the extent -+ 0.1,
    then centre and half extents, in f32."""
    off = np.float32(0.1)
    # (min over (p - 0.1) == min(p) - 0.1: f32 subtraction of a constant is monotone)
    lo = (np.asarray(pmin, np.float32) - off).astype(np.float32)
    hi = (np.asarray(pmax, np.float32) + off).astype(np.float32)
    two = np.float32(2.0)
    center = ((lo + hi).astype(np.float32) / two).astype(np.float32)
    half = ((hi - lo).astype(np.float32) / two).astype(np.float32)
    return (center - half).astype(np.float32), (center + half).astype(np.float32)


def random_gaussians_3d_seeded(n: int, seed: int = 0, chunk: int = 1 << 18, sh_degree: int = 3) -> PlanarGaussian3d:
    """planar_3d.rs:182-191 (distributions + field order), Philox stream, deterministic in (n, seed).  sh_degree < 3:
    the same cloud through `with_sh_degree` (the lower bands of the same draws, padding lanes zero)."""
    rng = np.random.Generator(np.random.Philox(seed))
    pos = np.empty((n, 4), np.float32)
    sh = np.empty((n, SH_COEFF_COUNT), np.float32)
    rot = np.empty((n, 4), np.float32)
    so = np.empty((n, 4), np.float32)
    for lo in range(0, n, chunk):
        hi = min(n, lo + chunk)
        u = rng.random((chunk, 59), dtype=np.float32)[: hi - lo]  # always draw whole chunks: stream is n-independent
        rot[lo:hi] = u[:, 0:4] * 2.0 - 1.0
        pos[lo:hi, 0:3] = u[:, 4:7] * 40.0 - 20.0
        pos[lo:hi, 3] = 1.0
        so[lo:hi, 0:3] = u[:, 7:10]
        so[lo:hi, 3] = u[:, 10] * 0.8
        sh[lo:hi] = u[:, 11:59] * 2.0 - 1.0
    cloud = PlanarGaussian3d(pos, sh, rot, so)
    return cloud if sh_degree == 3 else cloud.with_sh_degree(sh_degree)


def random_gaussians_3d(n: int) -> PlanarGaussian3d:
    """planar_3d.rs:170-180 (unseeded in the reference; seed 0 here so runs are reproducible)."""
    return random_gaussians_3d_seeded(n, 0)


SH_4D_COEFF_COUNT = 144  # src/material/spherindrical_harmonics.rs: SH-3 colour times time degree 2


@dataclasses.dataclass
class PlanarGaussian4d:
    """src/gaussian/formats/planar_4d.rs:38-51: the five planes `bgs_cloud_upload_4d` borrows."""
    position_visibility: np.ndarray     # (n, 4) f32: x, y, z, visibility
    spherindrical_harmonic: np.ndarray  # (n, 144) f32: SH-3 colour (0..47), cos(2 pi t) set (48..95), cos(4 pi t) set
    isotropic_rotations: np.ndarray     # (n, 8) f32: rotation (w, x, y, z), rotation_r (w, x, y, z); not normalised
    scale_opacity: np.ndarray           # (n, 4) f32: sx, sy, sz, opacity
    timestamp_timescale: np.ndarray     # (n, 4) f32: timestamp, timescale, pad, pad

    def __post_init__(self):
        for name, width in (("position_visibility", 4), ("spherindrical_harmonic", SH_4D_COEFF_COUNT),
                            ("isotropic_rotations", 8), ("scale_opacity", 4), ("timestamp_timescale", 4)):
            a = np.ascontiguousarray(getattr(self, name), dtype=np.float32)
            if a.ndim != 2 or a.shape[1] != width:
                raise ValueError(f"{name} must have shape (n, {width})")
            setattr(self, name, a)
        n = len(self.position_visibility)
        if not all(len(getattr(self, f.name)) == n for f in dataclasses.fields(self)):
            raise ValueError("planes disagree on n")

    def __len__(self) -> int:
        return len(self.position_visibility)

    def planes(self) -> tuple[np.ndarray, ...]:
        return tuple(getattr(self, f.name) for f in dataclasses.fields(self))

    def subset(self, n) -> "PlanarGaussian4d":
        """An int: the first n gaussians.  An index array: those gaussians, in that order."""
        idx = slice(0, n) if np.ndim(n) == 0 else np.asarray(n)
        return PlanarGaussian4d(*(a[idx] for a in self.planes()))

    def compute_aabb(self) -> tuple[np.ndarray, np.ndarray]:
        return compute_aabb(self.position_visibility)


def random_gaussians_4d_seeded(n: int, seed: int = 0, chunk: int = 1 << 16) -> PlanarGaussian4d:
    """planar_4d.rs:244-289 (distributions + field order: 144 coefficients U(-1,1); both rotations 8xU(-1,1),
    unnormalised; position 3xU(-20,20), visibility 1; scale 3xU(0,1), opacity U(0,0.8); timestamp U(0,1), timescale
    U(-1,1), pads 0), Philox stream, deterministic in (n, seed)."""
    rng = np.random.Generator(np.random.Philox(seed))
    planes = (np.empty((n, 4), np.float32), np.empty((n, SH_4D_COEFF_COUNT), np.float32), np.empty((n, 8), np.float32),
              np.empty((n, 4), np.float32), np.zeros((n, 4), np.float32))
    pos, sh, rot, so, tt = planes
    for lo in range(0, n, chunk):
        hi = min(n, lo + chunk)
        u = rng.random((chunk, 163), dtype=np.float32)[: hi - lo]  # always draw whole chunks: stream is n-independent
        sh[lo:hi] = u[:, 0:144] * 2.0 - 1.0
        rot[lo:hi] = u[:, 144:152] * 2.0 - 1.0
        pos[lo:hi, 0:3] = u[:, 152:155] * 40.0 - 20.0
        pos[lo:hi, 3] = 1.0
        so[lo:hi, 0:3] = u[:, 155:158]
        so[lo:hi, 3] = u[:, 158] * 0.8
        tt[lo:hi, 0] = u[:, 159]
        tt[lo:hi, 1] = u[:, 160] * 2.0 - 1.0
    return PlanarGaussian4d(*planes)


def test_model(seed: int = 0) -> PlanarGaussian3d:
    """planar_3d.rs:193-251: 8 corner gaussians at (+-0.5)^3 + a repeat of the first, shuffled SH."""
    rng = np.random.Generator(np.random.Philox(seed))
    base = rng.random(SH_COEFF_COUNT, dtype=np.float32) * 2.0 - 1.0
    pos, sh = [], []
    for x in (-0.5, 0.5):
        for y in (-0.5, 0.5):
            for z in (-0.5, 0.5):
                pos.append([x, y, z, 1.0])
                sh.append(rng.permutation(base))
    pos.append(pos[0]); sh.append(sh[0])
    n = len(pos)
    return PlanarGaussian3d(np.array(pos, np.float32), np.array(sh, np.float32),
                            np.tile(np.array([1, 0, 0, 0], np.float32), (n, 1)),
                            np.tile(np.array([0.125] * 4, np.float32), (n, 1)))
