"""Inputs of bgs_render_entities' tests (tests/test_oracle_entities.py, tests/test_gpu_entities.py): scene4d_cases' room
of 3D clouds and its 4D performer, listed twice, each entity with its own settings, so that splats of every blend kind
(quad-uv, conic, surfel) and of 4D clouds share tiles and list positions."""
from __future__ import annotations

import dataclasses

import bevy_gaussian_splatting_b200 as B
import scene4d_cases as S4
import scene_cases as SC

M, G, D = B.RasterizeMode, B.GaussianMode, B.DrawMode

# per entity: room clouds 0..3 (f32 deg 3, f16 deg 1, covariance deg 3, f32 deg 0), then the performer at two times
CASES = {
    # one of each blend kind among the 3D clouds, the performer as quad-uv and as conic
    "kinds": [dict(), dict(aabb=True), dict(), dict(gaussian_mode=G.Gaussian2d, aabb=True),
              dict(), dict(aabb=True)],
    # the same kinds with per-entity colour sources, draw modes and cutoffs
    "modes": [dict(rasterize_mode=M.Depth, draw_mode=D.HighlightSelected), dict(aabb=True, rasterize_mode=M.Normal),
              dict(rasterize_mode=M.Position, opacity_adaptive_radius=False),
              dict(gaussian_mode=G.Gaussian2d, aabb=True, draw_mode=D.Selected),
              dict(rasterize_mode=M.Velocity), dict(aabb=True, rasterize_mode=M.Depth)],
    # 2DGS with aabb beside the performer (bgs_render_scene_4d refuses this frame)
    "surfel_4d": [dict(gaussian_mode=G.Gaussian2d, aabb=True), dict(gaussian_mode=G.Gaussian2d, aabb=True),
                  dict(aabb=True), dict(gaussian_mode=G.Gaussian2d, aabb=True),
                  dict(rasterize_mode=M.Position), dict(aabb=True)],
    # Classification and OpticalFlow per entity, with their own num_classes, beside Color and Selected ones
    "classes": [dict(rasterize_mode=M.Classification, num_classes=3), dict(rasterize_mode=M.OpticalFlow, aabb=True),
                dict(), dict(gaussian_mode=G.Gaussian2d, rasterize_mode=M.Classification, num_classes=7),
                dict(rasterize_mode=M.Classification, num_classes=4), dict(rasterize_mode=M.OpticalFlow, draw_mode=D.Selected)],
    # every entity with the same settings: bgs_render_scene_4d's frame
    "agree": [dict()] * 6,
    "agree_aabb": [dict(aabb=True, rasterize_mode=M.Depth)] * 6,
}
TIMES = ((0.35, None), (0.8, SC.transform((0.4, 0.1, -0.3), 1.1, 0.9)))


def entities(case: str, n4: int = 5000):
    """[(cloud, layout or None for 4D, transform, CloudSettings)] of one case."""
    spec = CASES[case]
    out = []
    for (cloud, layout, _, tr, kw), over in zip(S4.room(), spec[:4]):
        out.append((cloud, layout, tr, B.CloudSettings(**{**kw, **over})))
    perf = S4.performer(n4, 9)
    for (t, tr), over in zip(TIMES, spec[4:]):
        st = S4.settings_4d(dataclasses.replace(B.CloudSettings(global_opacity=0.9), **over), t, -0.2, 1.1)
        out.append((perf, None, tr, st))
    return out


def kind(st: B.CloudSettings) -> int:
    """The blend kind of an entity's splats: 0 quad-uv, 1 conic, 2 surfel."""
    return 0 if not st.aabb else (2 if st.gaussian_mode == G.Gaussian2d else 1)


def oracle_entry(cloud, layout, u, st):
    """An entity as the scene4d / entity oracles list it."""
    if layout is None:
        return (cloud, u, (st.time_start, st.time_stop))
    return (SC.oracle_cloud(cloud, layout), u, layout == "cov")
