"""Inputs of bgs_render_views' tests (tests/test_gpu_views.py): view sets (a stereo pair, three views of different sizes
that the 16-pixel tile does not divide, six cube faces) around scene4d_cases' room, and entity mixes from entity_cases'
room and performer that reach each blend kernel a views frame launches:
  quad         raster_kernel<0, false, Z, false, ViewTable>  quad-uv entities: HighlightSelected, Classification, Position, 4D
  quad_box     raster_kernel<0, false, Z, true, ViewTable>   the same, every entity's overlay (the frame-wide flag)
  conic        raster_kernel<1, false, Z, false, ViewTable>  every entity 3DGS or 4D with aabb
  surfel       raster_kernel<2, false, Z, false, ViewTable>  every entity 2DGS with aabb (the room's f32 / f16 clouds)
  mixed        raster_kernel<4, false, Z, false, ViewTable>  entity_cases' "kinds": quad-uv, conic, surfel and 4D entities
  mixed_box    raster_kernel<4, false, Z, true, ViewTable>   the same, some entities with their overlay
  mixed_conic  raster_kernel<3, false, Z, false, ViewTable>  quad-uv and conic entities, Classification among them
(Z: with a depth buffer per view, or without.)  No entity is in Depth or OpticalFlow mode, which a views frame refuses."""
from __future__ import annotations

import dataclasses
import math

import bevy_gaussian_splatting_b200 as B
import scene4d_cases as S4
import scene_cases as SC

M, G, D = B.RasterizeMode, B.GaussianMode, B.DrawMode
ROOM = S4.ROOM_CENTRE

# per entity: room clouds 0..3 (f32 deg 3, f16 deg 1, covariance deg 3, f32 deg 0), then the performer at two times;
# None leaves the entity out
_AABB = dict(aabb=True)
_SURF = dict(gaussian_mode=G.Gaussian2d, aabb=True)
MIXES = {
    "quad": ([dict(draw_mode=D.HighlightSelected), dict(rasterize_mode=M.Classification, num_classes=3),
              dict(rasterize_mode=M.Position), dict(gaussian_mode=G.Gaussian2d), dict(), dict(draw_mode=D.Selected)], None, 0),
    "quad_box": ([dict(), dict(rasterize_mode=M.Position), dict(), dict(gaussian_mode=G.Gaussian2d), dict(), None], "frame", 0),
    "conic": ([_AABB, dict(aabb=True, rasterize_mode=M.Classification, num_classes=5), _AABB,
               dict(aabb=True, rasterize_mode=M.Normal), _AABB, None], None, 1),
    "surfel": ([_SURF, dict(_SURF, rasterize_mode=M.Position), None, dict(_SURF, draw_mode=D.HighlightSelected), None, None],
               None, 2),
    "mixed": ([dict(), _AABB, dict(), _SURF, dict(), _AABB], None, 4),
    "mixed_box": ([dict(), _AABB, dict(rasterize_mode=M.Position), _SURF, dict(), _AABB], [1, 0, 0, 1, 0, 1], 4),
    "mixed_conic": ([dict(rasterize_mode=M.Classification, num_classes=4), _AABB, dict(), dict(aabb=True, rasterize_mode=M.Normal),
                     None, None], None, 3),
}
TIMES = ((0.35, None), (0.8, SC.transform((0.4, 0.1, -0.3), 1.1, 0.9)))


def entities(mix: str, n4: int = 3000):
    """[(cloud, layout or None for 4D, transform, CloudSettings)] of one mix, its per-entity overlay bits, and whether the
    frame-wide overlay flag is set."""
    spec, flags, _ = MIXES[mix]
    out, bits = [], []
    for j, ((cloud, layout, _, tr, kw), over) in enumerate(zip(S4.room(), spec[:4])):
        if over is not None:
            out.append((cloud, layout, tr, B.CloudSettings(**{**kw, **over})))
            bits.append(flags[j] if isinstance(flags, list) else 0)
    perf = S4.performer(n4, 9)
    for j, ((t, tr), over) in enumerate(zip(TIMES, spec[4:]), 4):
        if over is not None:
            st = S4.settings_4d(dataclasses.replace(B.CloudSettings(global_opacity=0.9), **over), t, -0.2, 1.1)
            out.append((perf, None, tr, st))
            bits.append(flags[j] if isinstance(flags, list) else 0)
    return out, bits, flags == "frame"


def _around(eye, w, h, fov=math.pi / 4, target=ROOM, up=(0.0, 1.0, 0.0)):
    return B.perspective_view(eye, target, w, h, fov_y=fov, up=up)


def view_set(name: str) -> list[B.View]:
    if name == "stereo":   # two eyes 64 mm apart, looking straight at the room
        return [_around((x, 1.5, 3.0), 200, 120, target=(x, 1.5, -1.0)) for x in (-0.032, 0.032)]
    if name == "sizes":    # three cameras, three sizes, none a multiple of the tile size in both directions
        return [_around((0.0, 1.5, 3.0), 200, 120), _around((1.5, 2.2, 2.0), 97, 61), _around((-1.2, 1.0, 2.5), 33, 250)]
    if name == "cube":     # six 90-degree faces from a point at the room's front edge
        eye = (0.0, 1.5, 0.5)
        dirs = [((1, 0, 0), (0, 1, 0)), ((-1, 0, 0), (0, 1, 0)), ((0, 1, 0), (0, 0, 1)), ((0, -1, 0), (0, 0, 1)),
                ((0, 0, 1), (0, 1, 0)), ((0, 0, -1), (0, 1, 0))]
        return [_around(eye, 48, 48, math.pi / 2, tuple(e + d for e, d in zip(eye, dv)), up) for dv, up in dirs]
    raise KeyError(name)


VIEW_SETS = ("stereo", "sizes", "cube")
