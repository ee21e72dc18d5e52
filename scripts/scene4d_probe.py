"""What a dynamic 4D capture inside a static scan costs as one joint frame, against the per-entity composite and the scan
alone: bench.py's C3 cloud (6 M seeded gaussians, f16, global_scale 0.02) as the room, plus a seeded Gaussian4d cloud
of 500 k gaussians inside it (a box of half-side 2 in front of the camera, at time 0.5 of [0, 1]), at 1920x1080:

  (a) one bgs_render_scene_4d frame of both;
  (b) the per-entity composite: bgs_render of the room, then bgs_render_4d of the 4D cloud with
      BGS_FLAG_BLEND_OVER_TARGET (the reference's order when the 4D cloud is the nearer entity);
  (c) the room alone through bgs_render_scene.

    python scripts/scene4d_probe.py [--frames N] [--out FILE]

Each frame is synchronous into a device target; p50 and p90 of N frames after 5 of warm-up (host clock around a call
that ends in a device synchronise), and each frame's launch count.  Prints one JSON line with the card's name and
power limit beside the numbers.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bevy_gaussian_splatting_b200 as B  # noqa: E402
from bevy_gaussian_splatting_b200 import abi  # noqa: E402

W, H, N, SCALE, N4 = 1920, 1080, 6_000_000, 0.02, 500_000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, frames):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(frames):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return {"p50_ms": round(float(np.percentile(ts, 50)), 4), "p90_ms": round(float(np.percentile(ts, 90)), 4)}


def performer(n, seed=1):
    """n seeded Gaussian4d gaussians in a box of half-side 2 around (0, 1.5, -2), scales shrunk by 0.06."""
    c = B.random_gaussians_4d_seeded(n, seed)
    pos = c.position_visibility.copy()
    pos[:, :3] = pos[:, :3] * np.float32(2.0 / 20.0) + np.asarray((0.0, 1.5, -2.0), np.float32)
    so = c.scale_opacity.copy()
    so[:, :3] *= np.float32(0.06)
    return B.PlanarGaussian4d(pos, c.spherindrical_harmonic * np.float32(0.3), c.isotropic_rotations, so, c.timestamp_timescale)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "n_room": N, "n_4d": N4, "viewport": [W, H], "room_layout": "f16", "frames": a.frames}
    p = B.GaussianSplattingPlugin(0)
    lib, ctx = p._lib, p._ctx
    v = B.headless_view(W, H).to_abi()
    st = B.CloudSettings(global_scale=SCALE)
    st4 = B.CloudSettings(gaussian_mode=B.GaussianMode.Gaussian4d, time=0.5, time_start=0.0, time_stop=1.0)
    s, s4 = st.to_abi(), st4.to_abi()
    s4_over = st4.to_abi()
    s4_over.flags |= abi.BGS_FLAG_BLEND_OVER_TARGET
    room = p.add_cloud(B.random_gaussians_3d_seeded(N, 0), f16=True)
    h4 = p.add_cloud(performer(N4))
    u, u4 = p.cloud_uniform(st, None, room.aabb), p.cloud_uniform(st4, None, h4.aabb)
    out = torch.empty((H, W, 4), dtype=torch.uint8, device="cuda")
    code = abi.BGS_FORMAT_RGBA8_SRGB
    clouds = (C.c_void_p * 2)(room._h.value, h4._h.value)
    unis = (abi.bgs_cloud_uniform * 2)(u, u4)
    windows = (abi.bgs_time_window * 2)(abi.bgs_time_window(0.0, 1.0), abi.bgs_time_window(0.0, 1.0))

    def check(status):
        if status != abi.BGS_OK:
            raise RuntimeError(lib.bgs_last_error(ctx).decode())

    def joint():
        check(lib.bgs_render_scene_4d(ctx, clouds, unis, windows, 2, C.byref(v), C.byref(s), None, None, out.data_ptr(), code, 1))

    launches = {}

    def composite():
        check(lib.bgs_render(ctx, room._h, C.byref(v), C.byref(u), C.byref(s), out.data_ptr(), code, 1))
        launches["room"] = p.last_launch_count
        check(lib.bgs_render_4d(ctx, h4._h, C.byref(v), C.byref(u4), C.byref(s4_over), None, None, out.data_ptr(), code, 1,
                                C.c_float(0.0), C.c_float(1.0)))
        launches["4d"] = p.last_launch_count

    def room_alone():
        check(lib.bgs_render_scene(ctx, clouds, unis, 1, C.byref(v), C.byref(s), None, None, out.data_ptr(), code, 1))

    res["a_scene_4d"] = timed(joint, a.frames) | {"launches": p.last_launch_count, "n_visible": p.frame_stats().n_visible}
    res["b_composite"] = timed(composite, a.frames) | {"launches": launches["room"] + launches["4d"]}
    res["c_room_scene"] = timed(room_alone, a.frames) | {"launches": p.last_launch_count}
    res["a_over_b"] = round(res["a_scene_4d"]["p50_ms"] / res["b_composite"]["p50_ms"], 4)
    res["a_over_c"] = round(res["a_scene_4d"]["p50_ms"] / res["c_room_scene"]["p50_ms"], 4)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    p.destroy()


if __name__ == "__main__":
    main()
