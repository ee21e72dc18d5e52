"""Inputs of bgs_render_entities_aux's tests (tests/test_gpu_entities_aux.py): scene4d_cases' room of 3D clouds without
its covariance cloud (an aux frame refuses it), its first cloud listed a second time under another transform
(instancing), each entity with its own settings and overlay bit.

The cases reach every blend instantiation an aux frame can take; with the depth buffer on or off (the tests' other
parameter) they launch each kernel below once as given and once with ZTEST:
  quad              raster_kernel<0, true, Z, false, OneView>  every entity quad-uv (3DGS and 2DGS without aabb)
  quad_box          raster_kernel<0, true, Z, true, OneView>   the same, every entity with its overlay
  conic             raster_kernel<1, true, Z, false, OneView>  every entity 3DGS with aabb
  conic_box         raster_kernel<1, true, Z, true, OneView>
  surfel            raster_kernel<2, true, Z, false, OneView>  every entity 2DGS with aabb
  surfel_box        raster_kernel<2, true, Z, true, OneView>
  mixed             raster_kernel<3, true, Z, false, OneView>  quad-uv and conic entities
  mixed_box         raster_kernel<3, true, Z, true, OneView>   the same, two entities with their overlay
  mixed_surfel      raster_kernel<4, true, Z, false, OneView>  quad-uv, conic and surfel entities
  mixed_surfel_box  raster_kernel<4, true, Z, true, OneView>   the same, the surfel entity with its overlay
Colour sources differ per entity (Color, Depth, Normal, Position, Classification, OpticalFlow) and so do draw modes, so
the rgba frame and its Depth / Normal substitutes all differ."""
from __future__ import annotations

import dataclasses

import bevy_gaussian_splatting_b200 as B
import scene4d_cases as S4
import scene_cases as SC

M, G, D = B.RasterizeMode, B.GaussianMode, B.DrawMode

# entities: room clouds 0 (f32 deg 3), 1 (f16 deg 1), 3 (f32 deg 0), then cloud 0 again at INSTANCE
ROOM = (0, 1, 3, 0)
INSTANCE = SC.transform((0.5, -0.2, 0.3), 0.9, 0.6)

_QUAD = [dict(), dict(rasterize_mode=M.Depth, draw_mode=D.HighlightSelected),
         dict(gaussian_mode=G.Gaussian2d, rasterize_mode=M.Position), dict(rasterize_mode=M.Classification, num_classes=3)]
_CONIC = [dict(aabb=True), dict(aabb=True, rasterize_mode=M.Normal), dict(aabb=True, rasterize_mode=M.OpticalFlow),
          dict(aabb=True, rasterize_mode=M.Depth, draw_mode=D.Selected)]
_SURFEL = [dict(gaussian_mode=G.Gaussian2d, aabb=True), dict(gaussian_mode=G.Gaussian2d, aabb=True, rasterize_mode=M.Position),
           dict(gaussian_mode=G.Gaussian2d, aabb=True, rasterize_mode=M.Classification, num_classes=5),
           dict(gaussian_mode=G.Gaussian2d, aabb=True, draw_mode=D.HighlightSelected)]
_MIXED = [dict(), dict(aabb=True, rasterize_mode=M.Normal), dict(gaussian_mode=G.Gaussian2d, rasterize_mode=M.Classification,
                                                                  num_classes=4),
          dict(aabb=True, rasterize_mode=M.OpticalFlow)]
_MIXED_SURFEL = [dict(draw_mode=D.HighlightSelected), dict(aabb=True, rasterize_mode=M.Depth),
                 dict(gaussian_mode=G.Gaussian2d, aabb=True), dict(aabb=True, rasterize_mode=M.Classification, num_classes=2)]

# name -> (per-entity settings, per-entity overlay bits, blend mode of launch_raster)
CASES = {
    "quad": (_QUAD, [0, 0, 0, 0], 0), "quad_box": (_QUAD, [1, 1, 1, 1], 0),
    "conic": (_CONIC, [0, 0, 0, 0], 1), "conic_box": (_CONIC, [1, 1, 1, 1], 1),
    "surfel": (_SURFEL, [0, 0, 0, 0], 2), "surfel_box": (_SURFEL, [1, 1, 1, 1], 2),
    "mixed": (_MIXED, [0, 0, 0, 0], 3), "mixed_box": (_MIXED, [1, 1, 0, 0], 3),
    "mixed_surfel": (_MIXED_SURFEL, [0, 0, 0, 0], 4), "mixed_surfel_box": (_MIXED_SURFEL, [0, 0, 1, 0], 4),
}


def entities(case: str):
    """[(cloud, layout, transform, CloudSettings)] of one case, and its overlay bits."""
    spec, flags, _ = CASES[case]
    room = S4.room()
    out = []
    for j, (ri, over) in enumerate(zip(ROOM, spec)):
        cloud, layout, _, tr, kw = room[ri]
        out.append((cloud, layout, INSTANCE if j == 3 else tr, B.CloudSettings(**{**kw, **over})))
    return out, list(flags)


def with_mode(settings, mode):
    """Each entity's settings with rasterize_mode replaced by `mode` (what the aux frames equal)."""
    return [dataclasses.replace(st, rasterize_mode=mode) for st in settings]


def kinds(settings) -> set[int]:
    """The blend kinds among the entities: 0 quad-uv, 1 conic, 2 surfel."""
    return {0 if not st.aabb else (2 if st.gaussian_mode == G.Gaussian2d else 1) for st in settings}
