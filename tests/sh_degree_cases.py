"""Clouds stored at SH degree 0, 1 and 2 (include/bgs.h: K_d = (d + 1)^2 coefficients per channel, S_d = 4, 12, 28, 48
floats per gaussian) and the rules the tests restate in numpy:

* `rest_index`: where a ply's f_rest_i lands in an sh_d build (io/ply.rs:47-69, quirks kept);
* `colour`: the degree-d SH colour, 0.5 + sum over k < K_d of shc[k] basis_k(dir) sh[3k + c], then the sRGB decode;
* `embed48` / `embed24`: a degree-d SH plane as the first lanes (words) of a degree-3 one, the rest zero -- what the
  degree-3 oracles take.  Zero padding lanes make it `with_sh_degree(3)`, the cloud that renders like the degree-d one.
"""
from __future__ import annotations

import numpy as np

import bevy_gaussian_splatting_b200 as B
from bevy_gaussian_splatting_b200.gaussian import SH_WIDTHS, sh_bands

DEGREES = (0, 1, 2)
LAYOUTS = ("f32", "f16", "cov")

# spherical_harmonics.wgsl:3-20
SHC = np.array([0.28209479177387814, -0.4886025119029199, 0.4886025119029199, -0.4886025119029199,
                1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792,
                0.5462742152960396, -0.5900435899266435, 2.890611442640554, -0.4570457994644658,
                0.3731763325901154, -0.4570457994644658, 1.445305721320277, -0.5900435899266435])


def padding_lanes(d: int) -> list[int]:
    """Lanes 3 K_d .. S_d - 1: stored, never evaluated (lane 3 at degree 0, lane 27 at degree 2)."""
    return list(range(3 * sh_bands(d), SH_WIDTHS[d]))


def rest_index(i: int, d: int) -> int | None:
    """The SH lane f_rest_i is stored in by an sh_d build, or None when it is dropped."""
    k = sh_bands(d)
    channel = i // k
    coefficient = 1 if k == 1 else (i % (k - 1)) + 1
    idx = 3 * coefficient + channel
    return idx if idx < SH_WIDTHS[d] else None


def embed48(sh: np.ndarray) -> np.ndarray:
    out = np.zeros((len(sh), 48), np.float32)
    out[:, :sh.shape[1]] = sh
    return out


def embed24(words: np.ndarray) -> np.ndarray:
    out = np.zeros((len(words), 24), np.uint32)
    out[:, :words.shape[1]] = words
    return out


def basis(dirs: np.ndarray) -> np.ndarray:
    """(n, 16) SH-3 basis of unit directions (spherical_harmonics.wgsl:34-68), constants folded in, f64."""
    x, y, z = dirs[:, 0], dirs[:, 1], dirs[:, 2]
    xx, yy, zz = x * x, y * y, z * z
    b = np.stack([np.ones_like(x), y, z, x, x * y, y * z, 2 * zz - xx - yy, x * z, xx - yy, y * (3 * xx - yy), x * y * z,
                  y * (4 * zz - xx - yy), z * (2 * zz - 3 * xx - 3 * yy), x * (4 * zz - xx - yy), z * (xx - yy),
                  x * (xx - 3 * yy)], axis=1)
    return b * SHC


def colour(cloud: B.PlanarGaussian3d, eye, srgb: bool) -> np.ndarray:
    """(n, 3) Color-mode colour of each gaussian under an identity model, f64, at the cloud's own degree."""
    d = cloud.sh_degree
    k = sh_bands(d)
    dirs = cloud.position_visibility[:, :3].astype(np.float64) - np.asarray(eye, np.float64)
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    bs = basis(dirs)[:, :k]
    sh = cloud.spherical_harmonic.astype(np.float64)
    rgb = np.stack([0.5 + (bs * sh[:, c:3 * k:3]).sum(axis=1) for c in range(3)], axis=1)
    if srgb:
        rgb = np.where(rgb <= 0.04045, rgb / 12.92, ((rgb + 0.055) / 1.055) ** 2.4)
    return rgb


def labelled_cloud(n: int, seed: int, d: int) -> B.PlanarGaussian3d:
    """A seeded degree-d cloud whose visibility lanes hold class labels 1..4 (Classification reads them; DrawMode::All
    ignores them) and whose padding lanes are zero."""
    c = B.random_gaussians_3d_seeded(n, seed, sh_degree=d)
    c.position_visibility[:, 3] = np.random.default_rng(seed).integers(1, 5, n).astype(np.float32)
    return c


def with_padding_noise(cloud: B.PlanarGaussian3d, seed: int) -> B.PlanarGaussian3d:
    """The same cloud with non-zero values in its padding lanes (same values in every other lane)."""
    sh = cloud.spherical_harmonic.copy()
    lanes = padding_lanes(cloud.sh_degree)
    sh[:, lanes] = np.random.default_rng(seed).uniform(-4, 4, (len(sh), len(lanes))).astype(np.float32)
    return B.PlanarGaussian3d(cloud.position_visibility, sh, cloud.rotation, cloud.scale_opacity)
