"""What one frame of entities with their own settings costs: bench.py's C3 room (6 M seeded gaussians, f16, OBB,
global_scale 0.02) with a 500 k-gaussian 2DGS object drawn with aabb inside it, at 1920x1080, rendered

  (a) as one bgs_render_entities frame (room quad-uv, object surfel: the mixed-kind blend);
  (b) the room as a bgs_render_scene frame, then the object as a bgs_render with BGS_FLAG_BLEND_OVER_TARGET (what an
      app does without per-entity settings);
  (c) the room alone (bgs_render_scene).

    python scripts/entities_probe.py [--frames N] [--out FILE]

Each frame is synchronous into a device target; p50 and p90 of N frames after 5 of warm-up (host clock around a call
that ends in a device synchronise), the launch count, and the blend stage's time (bgs_stage_times_us[4]) of (a) and (c):
raster_mixed_kernel<4> against raster_kernel<0> over the same room.  Prints one JSON line with the card's name and power
limit beside the numbers.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bevy_gaussian_splatting_b200 as B  # noqa: E402
from bevy_gaussian_splatting_b200 import abi  # noqa: E402
from bevy_gaussian_splatting_b200.plugin import entity_settings  # noqa: E402
from scripts.scene_probe import card, timed  # noqa: E402

W, H, N, N_OBJ, SCALE = 1920, 1080, 6_000_000, 500_000, 0.02


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "n_room": N, "n_object": N_OBJ, "viewport": [W, H], "frames": a.frames}
    p = B.GaussianSplattingPlugin(0)
    lib, ctx = p._lib, p._ctx
    v = B.headless_view(W, H).to_abi()
    room_st = B.CloudSettings(global_scale=SCALE)
    obj_st = B.CloudSettings(global_scale=SCALE, gaussian_mode=B.GaussianMode.Gaussian2d, aabb=True)
    room = p.add_cloud(B.random_gaussians_3d_seeded(N, 0), f16=True)
    obj = p.add_cloud(B.random_gaussians_3d_seeded(N_OBJ, 1))
    m = np.diag([0.3, 0.3, 0.3, 1.0]).astype(np.float32)   # the object: a third of the room's extent, inside it
    m[:3, 3] = (0.0, 1.0, 0.0)
    tr = B.CloudTransform(m)
    ur, uo = p.cloud_uniform(room_st, None, room.aabb), p.cloud_uniform(obj_st, tr, obj.aabb)
    s_room, s_obj = room_st.to_abi(), obj_st.to_abi()
    s_room.flags |= abi.BGS_FLAG_NO_CHUNKS
    s_obj.flags |= abi.BGS_FLAG_BLEND_OVER_TARGET
    out = torch.empty((H, W, 4), dtype=torch.uint8, device="cuda")
    code = abi.BGS_FORMAT_RGBA8_SRGB
    clouds2 = (C.c_void_p * 2)(room._h.value, obj._h.value)
    unis2 = (abi.bgs_cloud_uniform * 2)(ur, uo)
    ents2 = (abi.bgs_entity_settings * 2)(entity_settings(room_st), entity_settings(obj_st))
    clouds1 = (C.c_void_p * 1)(room._h.value)
    unis1 = (abi.bgs_cloud_uniform * 1)(ur)

    def check(status):
        if status != abi.BGS_OK:
            raise RuntimeError(lib.bgs_last_error(ctx).decode())

    def entities():
        check(lib.bgs_render_entities(ctx, clouds2, unis2, ents2, 2, C.byref(v), C.byref(s_room), None, None, out.data_ptr(), code, 1))

    def room_alone():
        check(lib.bgs_render_scene(ctx, clouds1, unis1, 1, C.byref(v), C.byref(s_room), None, None, out.data_ptr(), code, 1))

    def composite():
        room_alone()
        check(lib.bgs_render(ctx, obj._h, C.byref(v), C.byref(uo), C.byref(s_obj), out.data_ptr(), code, 1))

    res["a_entities"] = timed(entities, a.frames) | {"launches": p.last_launch_count,
                                                     "blend_us": round(float(p.stage_times_us()[4]), 1)}
    res["b_scene_then_blend_over"] = timed(composite, a.frames)
    res["c_room_alone"] = timed(room_alone, a.frames) | {"launches": p.last_launch_count,
                                                         "blend_us": round(float(p.stage_times_us()[4]), 1)}
    res["a_over_b"] = round(res["a_entities"]["p50_ms"] / res["b_scene_then_blend_over"]["p50_ms"], 4)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    p.destroy()


if __name__ == "__main__":
    main()
