"""Inputs of bgs_render_scene_4d's tests (tests/test_oracle_scene_4d.py, tests/test_gpu_scene_4d.py): a seeded Gaussian4d
"performer" placed inside scene_cases' room of 3D clouds, its settings, and the colour bound of its SH records."""
from __future__ import annotations

import dataclasses

import numpy as np

import bevy_gaussian_splatting_b200 as B
import scene_cases as SC

f32 = np.float32
ROOM_CENTRE = (0.0, 1.5, -1.0)


def performer(n: int, seed: int, centre=ROOM_CENTRE, spread: float = 0.9, scale: float = 0.06) -> B.PlanarGaussian4d:
    """n Gaussian4d gaussians in a box of half-side `spread` around `centre`; timescales in [0.2, 1) so that some are
    masked at every time and some are not; visibility a mix of 0, 1 and class labels for the draw and class modes."""
    c = B.random_gaussians_4d_seeded(n, seed)
    rng = np.random.default_rng(seed)
    pos = c.position_visibility.copy()
    pos[:, :3] = pos[:, :3] * f32(spread / 20.0) + np.asarray(centre, f32)
    pos[:, 3] = rng.choice(np.array([0.0, 1.0, 2.0, 3.5], f32), n)
    so = c.scale_opacity.copy()
    so[:, :3] *= f32(scale)
    tt = c.timestamp_timescale.copy()
    tt[:, 1] = np.where(tt[:, 1] < 0, f32(-1.0), f32(1.0)) * (f32(0.2) + np.abs(tt[:, 1]) * f32(0.8))
    return B.PlanarGaussian4d(pos, c.spherindrical_harmonic * f32(0.3), c.isotropic_rotations, so, tt)


def settings_4d(base: B.CloudSettings, time: float, time_start: float = 0.0, time_stop: float = 1.0, **kw) -> B.CloudSettings:
    """`base` as a 4D entity's settings at `time` in [time_start, time_stop]."""
    return dataclasses.replace(base, gaussian_mode=B.GaussianMode.Gaussian4d, time=time, time_start=time_start,
                               time_stop=time_stop, **kw)


def room(seed: int = 40):
    """[(cloud, layout, sh_degree, transform, settings overrides)]: f32, f16 and covariance clouds of several SH degrees
    around ROOM_CENTRE, with their own transforms, scales, opacities and colour spaces."""
    spec = [("f32", 3, SC.transform(), dict()),
            ("f16", 1, SC.transform((0.3, 0.1, 0.2), 1.2, 0.7), dict(global_scale=1.3, global_opacity=0.8)),
            ("cov", 3, SC.transform((-0.4, 0.0, -0.2)), dict(color_space=B.GaussianColorSpace.LinRec709Display)),
            ("f32", 0, SC.transform((0.1, -0.3, 0.4), 0.8, -0.5), dict(global_opacity=0.6))]
    return [(SC.cloud_in_box(3000, seed + j, centre=ROOM_CENTRE, half=1.2, scale=0.08, sh_degree=d), layout, d, tr, kw)
            for j, (layout, d, tr, kw) in enumerate(spec)]


def sh_bound(cloud: B.PlanarGaussian4d, ids) -> np.ndarray:
    """|colour - oracle colour| bound of a 4D record's SH colour (test_gpu_temporal's): 2e-5 of the SH sums' magnitude
    (basis terms <= 3 each), x 2.4 for the sRGB decode."""
    mag = f32(0.5) + 3.0 * np.abs(cloud.spherindrical_harmonic[ids]).reshape(-1, 48, 3).sum(1)
    return 2.4 * 2e-5 * mag + 1e-6


def drawn(records: np.ndarray) -> np.ndarray:
    """Records (n, 12) with a non-empty bbox."""
    bb = records[:, 6:8].view(np.uint32)
    return ((bb[:, 0] & 0xFFFF) <= (bb[:, 0] >> 16)) & ((bb[:, 1] & 0xFFFF) <= (bb[:, 1] >> 16))
