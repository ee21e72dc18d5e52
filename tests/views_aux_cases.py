"""Inputs of bgs_render_views_aux's tests (tests/test_gpu_views_aux.py): entity_aux_cases' mixes with their OpticalFlow
entity swapped for another mode (a views frame refuses OpticalFlow), seen through views_cases' view sets, and a small
cloud whose views cover the Depth range's edge cases.

Each mix reaches one blend kernel of bgs_render_views_aux; with the per-view depth buffers on or off (the tests' other
parameter) it launches it once as given and once with ZTEST:
  quad              raster_kernel<0, true, Z, false, ViewTable>  every entity quad-uv; a Depth entity
  quad_box          raster_kernel<0, true, Z, true, ViewTable>   the same, every entity with its overlay
  conic             raster_kernel<1, true, Z, false, ViewTable>  every entity 3DGS with aabb; a Depth entity
  conic_box         raster_kernel<1, true, Z, true, ViewTable>
  surfel            raster_kernel<2, true, Z, false, ViewTable>  every entity 2DGS with aabb
  surfel_box        raster_kernel<2, true, Z, true, ViewTable>
  mixed             raster_kernel<3, true, Z, false, ViewTable>  quad-uv and conic entities; a Depth entity
  mixed_box         raster_kernel<3, true, Z, true, ViewTable>   the same, two entities with their overlay
  mixed_surfel      raster_kernel<4, true, Z, false, ViewTable>  quad-uv, conic and surfel entities; a Depth entity
  mixed_surfel_box  raster_kernel<4, true, Z, true, ViewTable>   the same, the surfel entity with its overlay
Every mix's depth frames are over each view's own range, whether or not an entity is in Depth mode."""
from __future__ import annotations

import math

import numpy as np

import bevy_gaussian_splatting_b200 as B
import entity_aux_cases as EA

M = B.RasterizeMode

# the entity (by case) that entity_aux_cases puts in OpticalFlow mode, and what it becomes here
_SWAP = {"conic": (2, dict(aabb=True, rasterize_mode=M.Classification, num_classes=3)),
         "conic_box": (2, dict(aabb=True, rasterize_mode=M.Classification, num_classes=3)),
         "mixed": (3, dict(aabb=True, rasterize_mode=M.Depth)),
         "mixed_box": (3, dict(aabb=True, rasterize_mode=M.Depth))}
CASES = {name: mode for name, (_, _, mode) in EA.CASES.items()}


def entities(case: str):
    """[(cloud, layout, transform, CloudSettings)] of one mix, and its overlay bits."""
    listed, flags = EA.entities(case)
    if case in _SWAP:
        j, over = _SWAP[case]
        cloud, layout, tr, _ = listed[j]
        kw = {f: getattr(listed[j][3], f) for f in ("global_scale", "global_opacity", "color_space")}
        listed[j] = (cloud, layout, tr, B.CloudSettings(**{**kw, **over}))
    assert all(st.rasterize_mode != M.OpticalFlow for _, _, _, st in listed)
    return listed, flags


# ---- the Depth range's edge cases: seven gaussians around the origin and one at (20, 0, 0)
FAR = (20.0, 0.0, 0.0)


def edge_cloud(n_near: int = 7, seed: int = 5) -> B.PlanarGaussian3d:
    c = B.random_gaussians_3d_seeded(n_near + 1, seed, sh_degree=0)
    pos = c.position_visibility.copy()
    pos[:n_near, :3] = pos[:n_near, :3] * np.float32(0.3 / 20.0)
    pos[n_near, :3] = FAR
    pos[:, 3] = 1.0
    so = c.scale_opacity.copy()
    so[:, :3] *= np.float32(0.05)
    so[:, 3] = np.maximum(so[:, 3], 0.5)
    return B.PlanarGaussian3d(pos, c.spherical_harmonic, c.rotation, so)


def single_cloud() -> B.PlanarGaussian3d:
    """One gaussian at the origin (an entity list of one: its Depth colours are black)."""
    c = edge_cloud(0)
    c.position_visibility[0, :3] = 0.0
    return c


def edge_views(w: int = 64, h: int = 48) -> dict[str, B.View]:
    return {
        "most": B.perspective_view((0.0, 0.0, 5.0), (0.0, 0.0, 0.0), w, h),                    # the seven near ones
        "all": B.perspective_view((10.0, 0.0, 60.0), (10.0, 0.0, 0.0), w, h),                  # nothing culled
        "one": B.perspective_view((20.0, 0.0, 3.0), FAR, w, h, fov_y=math.pi / 8),             # exactly the far one
        "none": B.perspective_view((0.0, 0.0, 5.0), (0.0, 0.0, 10.0), w, h),                   # looking away: 0 visible
        "side": B.perspective_view((3.0, 1.0, 4.0), (0.0, 0.0, 0.0), w, h),
    }
