"""What one joint frame of several clouds costs against one cloud and against the per-entity composite: bench.py's C3
cloud (6 M seeded gaussians, f16, global_scale 0.02) at 1920x1080, rendered

  (a) whole, through bgs_render;
  (b) split into K contiguous subsets (bgs_cloud_subset in index mode), through one bgs_render_scene;
  (c) the same K subsets as K bgs_render calls, far first, each after the first with BGS_FLAG_BLEND_OVER_TARGET (the
      reference's per-entity order).

    python scripts/scene_probe.py [--frames N] [--mode Color|...|Classification] [--ks 2,8,64] [--out FILE]

Each frame is synchronous into a device target; p50 and p90 of N frames after 5 of warm-up (host clock around a call
that ends in a device synchronise), the p50 of the projection stage (bgs_stage_times_us()[2], device events) and the
frame's launch count.  --mode draws every frame in that RasterizeMode (default Color).  Also checks that (b)'s frame is
byte-identical to (a)'s.  Prints one JSON line with the card's name and power limit beside the numbers.
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

W, H, N, SCALE = 1920, 1080, 6_000_000, 0.02
KS = (2, 8, 64)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, frames, plugin=None):
    """p50 / p90 of `frames` calls of fn; with `plugin`, also the p50 of its last frame's projection stage."""
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    ts, proj = [], []
    for _ in range(frames):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
        if plugin is not None:
            proj.append(float(plugin.stage_times_us()[2]))
    r = {"p50_ms": round(float(np.percentile(ts, 50)), 4), "p90_ms": round(float(np.percentile(ts, 90)), 4)}
    if plugin is not None:
        r["proj_us_p50"] = round(float(np.percentile(proj, 50)), 2)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--mode", default="Color", choices=[m.name for m in B.RasterizeMode if m <= B.RasterizeMode.Classification])
    ap.add_argument("--ks", default=",".join(map(str, KS)))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "n": N, "viewport": [W, H], "layout": "f16", "frames": a.frames, "mode": a.mode}
    p = B.GaussianSplattingPlugin(0)
    lib, ctx = p._lib, p._ctx
    view = B.headless_view(W, H)
    v = view.to_abi()
    st = B.CloudSettings(global_scale=SCALE, rasterize_mode=B.RasterizeMode[a.mode])
    s = st.to_abi()
    s_over = st.to_abi()
    s_over.flags |= abi.BGS_FLAG_BLEND_OVER_TARGET
    cloud = B.random_gaussians_3d_seeded(N, 0)
    h = p.add_cloud(cloud, f16=True)
    u = p.cloud_uniform(st, None, h.aabb)
    out = torch.empty((H, W, 4), dtype=torch.uint8, device="cuda")
    code = abi.BGS_FORMAT_RGBA8_SRGB

    def check(status):
        if status != abi.BGS_OK:
            raise RuntimeError(lib.bgs_last_error(ctx).decode())

    def whole():
        check(lib.bgs_render(ctx, h._h, C.byref(v), C.byref(u), C.byref(s), out.data_ptr(), code, 1))

    res["a_whole"] = timed(whole, a.frames, p) | {"launches": p.last_launch_count}
    ref = out.clone()
    cam = np.asarray(view.to_abi().world_position[:3], np.float32)
    for k in map(int, a.ks.split(",")):
        cuts = np.linspace(0, N, k + 1).astype(np.int64)
        parts = [p.subset(h, np.arange(cuts[j], cuts[j + 1])) for j in range(k)]
        clouds = (C.c_void_p * k)(*[q._h.value for q in parts])
        unis = (abi.bgs_cloud_uniform * k)(*([u] * k))
        far_first = sorted(range(k), key=lambda j: -float(np.linalg.norm(
            cloud.position_visibility[cuts[j]:cuts[j + 1], :3].mean(0) - cam)))

        def scene():
            check(lib.bgs_render_scene(ctx, clouds, unis, k, C.byref(v), C.byref(s), None, None, out.data_ptr(), code, 1))

        def chain():
            for i, j in enumerate(far_first):
                check(lib.bgs_render(ctx, parts[j]._h, C.byref(v), C.byref(u), C.byref(s_over if i else s), out.data_ptr(), code, 1))

        r = {"b_scene": timed(scene, a.frames, p) | {"launches": p.last_launch_count}}
        r["b_identical_to_a"] = bool(torch.equal(out, ref))
        r["c_chain"] = timed(chain, a.frames)
        r["b_over_a"] = round(r["b_scene"]["p50_ms"] / res["a_whole"]["p50_ms"], 4)
        r["b_over_c"] = round(r["b_scene"]["p50_ms"] / r["c_chain"]["p50_ms"], 4)
        res[f"K{k}"] = r
        for q in parts:
            q.destroy()
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    p.destroy()


if __name__ == "__main__":
    main()
