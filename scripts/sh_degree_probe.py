"""What the SH degree of a resident cloud costs: 1 M and 6 M seeded gaussians (random_gaussians_3d_seeded, seed 0, the
lower degrees through its sh_degree argument), f32 and f16, SH degree 0..3, 1920x1080, Color mode, global_scale 0.02
(bench.py's C3 settings).

    python scripts/sh_degree_probe.py [--frames K] [--out FILE]

Per (n, layout, degree): the projection stage of one synchronous frame (bgs_stage_times_us[2], CUDA events, median of
10), ms per frame in bench.py's loop (consecutive frames alternating between three contexts, every frame queued; host
clock around K frames and the final syncs, median of 3 blocks), the resident bytes per gaussian the layout table gives
(16 B position plane + the block) and the device memory one upload took (cudaMemGetInfo before and after, so other work
on the card shows up in it).  Prints one JSON line with the card's name and power limit beside the numbers.
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

W, H, SCALE, CTX = 1920, 1080, 0.02, 3
SIZES = (1_000_000, 6_000_000)
BLOCK_BYTES = {"f32": (64, 128, 256, 256), "f16": (64, 64, 128, 128)}   # include/bgs.h


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def measure(plugins, cloud, f16, view, s, frames):
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    handles = [plugins[0].add_cloud(cloud, f16=f16)]
    torch.cuda.synchronize()
    used = free0 - torch.cuda.mem_get_info()[0]
    handles += [p.add_cloud(cloud, f16=f16) for p in plugins[1:]]
    p0, h0 = plugins[0], handles[0]
    stage = []
    for i in range(15):
        p0.render_view(h0, s, view, to_host=False)
        if i >= 5:
            stage.append(p0.stage_times_us())
    stage = np.median(np.array(stage), axis=0)
    n_vis = int(p0.frame_stats().n_visible)
    for p, h in zip(plugins, handles):   # warm the queued path
        p.render_view(h, s, view, to_host=False, asynchronous=True)
    for p in plugins:
        p.sync()
    blocks = []
    for _ in range(3):
        t0 = time.perf_counter()
        for k in range(frames):
            plugins[k % CTX].render_view(handles[k % CTX], s, view, to_host=False, asynchronous=True)
        for p in plugins:
            p.sync()
        blocks.append((time.perf_counter() - t0) * 1e3 / frames)
    for h in handles:
        h.destroy()
    return {"projection_us": round(float(stage[2]), 2), "stage_us": [round(float(x), 2) for x in stage],
            "ms_per_frame_3_in_flight": round(float(np.median(blocks)), 4), "blocks_ms": [round(b, 4) for b in blocks],
            "n_visible": n_vis, "upload_device_bytes_per_gaussian": round(used / len(cloud), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    view = B.headless_view(W, H)
    s = B.CloudSettings(global_scale=SCALE)
    plugins = [B.GaussianSplattingPlugin(0) for _ in range(CTX)]
    res = {"card_before": card(), "width": W, "height": H, "global_scale": SCALE, "frames": a.frames, "runs": []}
    for n in SIZES:
        full = B.random_gaussians_3d_seeded(n, 0)
        for layout in ("f32", "f16"):
            for d in (0, 1, 2, 3):
                cloud = full if d == 3 else full.with_sh_degree(d)
                r = measure(plugins, cloud, layout == "f16", view, s, a.frames)
                r.update(n=n, layout=layout, sh_degree=d, resident_bytes_per_gaussian=16 + BLOCK_BYTES[layout][d])
                print(json.dumps(r), flush=True)
                res["runs"].append(r)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    for p in plugins:
        p.destroy()


if __name__ == "__main__":
    main()
