"""Host-side mirror of the reference's per-cloud configuration surface.

Names, defaults and meaning follow src/gaussian/settings.rs:6-133 (enums + CloudSettings) and
src/render/mod.rs:698-760 (ShaderDefines: the radix pass plan).  Only what the forward splat path
reads is carried across the C ABI (`to_abi`); the rest is kept so user code reads the same.
"""
from __future__ import annotations

import dataclasses
import enum
from typing import Optional

import numpy as np

from . import abi


class DrawMode(enum.IntEnum):  # settings.rs:6-12
    All = 0
    Selected = 1
    HighlightSelected = 2


class GaussianMode(enum.IntEnum):  # settings.rs:17-22
    Gaussian2d = 0
    Gaussian3d = 1
    Gaussian4d = 2       # PlanarGaussian4d clouds, through bgs_render_4d


class RasterizeMode(enum.IntEnum):  # settings.rs:38-48
    Color = 0
    Depth = 1
    Normal = 2
    Position = 3
    Classification = 4   # the hue of class vis - 2 from the visibility lane, CloudSettings.num_classes hues
    OpticalFlow = 5      # camera motion since the previous view (render_view's previous_view / delta_time)
    Velocity = 6         # Gaussian4d only: each splat's velocity at CloudSettings.time


class RadixSortDepthBits(enum.IntEnum):  # settings.rs:50-77
    Bits16 = 16
    Bits24 = 24
    Bits32 = 32

    def bits(self) -> int:
        return int(self)


class GaussianColorSpace(enum.IntEnum):  # settings.rs:79-84
    SrgbRec709Display = 0
    LinRec709Display = 1


class PlaybackMode(enum.IntEnum):  # settings.rs:24-36
    Loop = 0
    Once = 1
    Sin = 2
    Still = 3


class SortMode(enum.IntEnum):  # src/sort/mod.rs:46-74; only Radix exists here (no CPU fallback)
    Radix = 0


@dataclasses.dataclass
class ShaderDefines:
    """The radix pass plan (src/render/mod.rs:698-760)."""

    radix_bits_per_digit: int
    radix_digit_places: int
    radix_key_shift: int
    radix_base: int

    @staticmethod
    def for_radix_depth_bits(bits: RadixSortDepthBits) -> "ShaderDefines":
        radix_bits_per_digit = 8
        return ShaderDefines(
            radix_bits_per_digit=radix_bits_per_digit,
            radix_digit_places=RadixSortDepthBits(bits).bits() // radix_bits_per_digit,
            radix_key_shift=32 - RadixSortDepthBits(bits).bits(),
            radix_base=1 << radix_bits_per_digit,
        )

    def radix_initial_parity(self) -> int:
        return self.radix_digit_places % 2


@dataclasses.dataclass
class SparseSelect:
    """src/query/sparse.rs:24-38, same field names and defaults: select the gaussians with fewer than
    `neighbor_threshold` gaussians (themselves included) within `radius` -- the floater filter
    (`GaussianSplattingPlugin.select_sparse`)."""

    radius: float = 0.05
    neighbor_threshold: int = 3


@dataclasses.dataclass
class CloudSettings:
    """src/gaussian/settings.rs:90-133, same field names and defaults."""

    aabb: bool = False
    global_opacity: float = 1.0
    global_scale: float = 1.0
    opacity_adaptive_radius: bool = True
    visualize_bounding_box: bool = False
    sort_mode: SortMode = SortMode.Radix
    radix_sort_depth_bits: RadixSortDepthBits = RadixSortDepthBits.Bits32
    draw_mode: DrawMode = DrawMode.All
    gaussian_mode: GaussianMode = GaussianMode.Gaussian3d
    rasterize_mode: RasterizeMode = RasterizeMode.Color
    color_space: GaussianColorSpace = GaussianColorSpace.SrgbRec709Display
    num_classes: int = 1
    time: float = 0.0
    # this repo's extension: sort all N entries like the reference instead of compacting first
    sort_all: bool = False
    # this repo's extension: front-to-back binning rounds (BGS_FLAG_CHUNKS): None = library's choice from the last
    # frame's footprint statistics, True = always, False = never (the tile debug hooks need a one-round frame)
    binning_rounds: Optional[bool] = None
    # the interpolation window (settings.rs:106-107, 128-129): `GaussianSplattingPlugin.interpolate` blends at
    # (time - time_start) / (time_stop - time_start).  Last, so positional construction keeps its meaning
    time_start: float = 0.0
    time_stop: float = 1.0
    # playback of a Gaussian4d cloud (settings.rs:110-111): how `playback_update` advances `time`
    time_scale: float = 1.0
    playback_mode: PlaybackMode = PlaybackMode.Still

    def to_abi(self) -> abi.bgs_settings:
        return abi.bgs_settings(
            gaussian_mode=int(self.gaussian_mode),
            rasterize_mode=int(self.rasterize_mode),
            aabb=int(bool(self.aabb)),
            opacity_adaptive_radius=int(bool(self.opacity_adaptive_radius)),
            draw_mode=int(self.draw_mode),
            radix_sort_depth_bits=int(self.radix_sort_depth_bits),
            flags=(abi.BGS_FLAG_SORT_ALL if self.sort_all else 0)
            | (0 if self.binning_rounds is None else (abi.BGS_FLAG_CHUNKS if self.binning_rounds else abi.BGS_FLAG_NO_CHUNKS))
            | (abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX if self.visualize_bounding_box else 0),
            reserved=0,
        )


def playback_update(settings: CloudSettings, delta_secs: float, elapsed_secs: float) -> None:
    """settings.rs:145-191, the reference's playback_update for one cloud, in f32 as there: nothing when time_scale is
    0 or the mode is Still, or in Once mode once time >= time_stop; Loop and Once add delta_secs * time_scale (Loop
    then wraps to time_start past time_stop; Once is not clamped); Sin sets time = time_start + (time_stop -
    time_start) * (sin(time_scale * elapsed_secs * 2 * PI) + 1) / 2.  np.sin of an f32 stands for Rust's f32 sin."""
    f = np.float32
    time, start, stop, scale = f(settings.time), f(settings.time_start), f(settings.time_stop), f(settings.time_scale)
    mode = PlaybackMode(settings.playback_mode)
    if scale == 0 or mode == PlaybackMode.Still or (mode == PlaybackMode.Once and time >= stop):
        return
    if mode in (PlaybackMode.Loop, PlaybackMode.Once):
        time = f(time + f(f(delta_secs) * scale))
        if mode == PlaybackMode.Loop and time > stop:
            time = start
    else:
        theta = f(scale * f(elapsed_secs))
        y = np.sin(f(f(theta * f(2.0)) * f(np.pi)), dtype=np.float32)
        time = f(start + f(f(f(stop - start) * f(y + f(1.0))) / f(2.0)))
    settings.time = float(time)
