"""What the depth test costs on the benchmarked frame (bench.py's C3: 6 M f16 gaussians, 1920x1080, global_scale 0.02),
three contexts in flight.

    python scripts/depth_probe.py [--frames K] [--out FILE]

Scene buffers: none (bgs_render), a zero (cleared reverse-Z) buffer, a plane in front of the cloud (depth 1.0) over the
left half of the screen, and the same plane over all of it.  Per buffer: ms per frame over K queued frames (scenarios
alternate round by round, so drift of the card's clock spreads over all of them), the blend stage of one synchronous
frame (bgs_stage_times_us, CUDA events) and splat_depth_kernel's time (torch.profiler's CUDA activity, in a run of its
own).  Prints one JSON line with the card's name and power limit beside the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bevy_gaussian_splatting_b200 as B  # noqa: E402

W, H, N, SCALE, CTX = 1920, 1080, 6_000_000, 0.02, 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    cloud = B.random_gaussians_3d_seeded(N, 0)
    view = B.headless_view(W, H)
    s = B.CloudSettings(global_scale=SCALE)
    ps = [B.GaussianSplattingPlugin(0) for _ in range(CTX)]
    h = ps[0].add_cloud(cloud, f16=True)
    half = torch.zeros((H, W), dtype=torch.float32, device="cuda")
    half[:, : W // 2] = 1.0
    scenes = {"none": None, "zero": torch.zeros((H, W), dtype=torch.float32, device="cuda"), "half_plane": half,
              "full_plane": torch.ones((H, W), dtype=torch.float32, device="cuda")}

    def frame(p, z, queued=True):
        p.render_view(h, s, view, fmt="rgba8_srgb", to_host=False, asynchronous=queued, scene_depth=z)

    for name, z in scenes.items():   # warm every path (and the hints) before timing
        for p in ps:
            for _ in range(3):
                frame(p, z, queued=False)
    ms = {k: [] for k in scenes}
    for _ in range(a.rounds):
        for name, z in scenes.items():
            for _ in range(2 * CTX):
                frame(ps[_ % CTX], z)
            for p in ps:
                assert p.sync()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(a.frames):
                frame(ps[i % CTX], z)
            for p in ps:
                assert p.sync()
            torch.cuda.synchronize()
            ms[name].append((time.perf_counter() - t0) * 1e3 / a.frames)
    blend_us = {}
    for name, z in scenes.items():
        st = []
        for _ in range(10):
            frame(ps[0], z, queued=False)
            st.append(ps[0].stage_times_us())
        blend_us[name] = round(float(np.median([x[4] for x in st])), 1)
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            frame(ps[0], scenes["zero"], queued=False)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if "splat_depth_kernel" in e.key or "raster" in e.key:
            kern[e.key.split("(")[0][:60]] = round(e.device_time_total / max(e.count, 1), 1)
    res = {"probe": "depth_test", "card": card(), "workload": f"C3: {N} f16, {W}x{H}, global_scale {SCALE}, {CTX} contexts in flight",
           "ms_per_frame": {k: [round(v, 4) for v in vs] for k, vs in ms.items()},
           "ms_per_frame_median": {k: round(float(np.median(vs)), 4) for k, vs in ms.items()},
           "blend_stage_us_sync": blend_us, "kernel_us_zero_buffer": kern}
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
