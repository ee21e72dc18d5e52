"""What a Gaussian4d frame costs: 2 M seeded 4D gaussians (random_gaussians_4d_seeded), 1920x1080, Color mode,
global_scale 0.02, at three times chosen so that different fractions of the cloud pass the time mask.

    python scripts/temporal_probe.py [--frames K] [--out FILE]

Per time: the fraction of the cloud drawn (n_visible records with a non-empty bbox over n), ms per frame one at a time
(synchronous frames, host clock around each completed frame) and with three contexts in flight (queued frames, host
clock around K frames and the final syncs), and the projection stage of one synchronous frame (bgs_stage_times_us,
CUDA events).  Prints one JSON line with the card's name and power limit beside the numbers.
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

import bevy_gaussian_splatting_b200 as B  # noqa: E402

W, H, N, SCALE, CTX = 1920, 1080, 2_000_000, 0.02, 3
TIMES = (0.5, 1.5, 3.0)   # inside the timestamps' [0, 1) span, past it, further past it


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    cloud = B.random_gaussians_4d_seeded(N, 0)
    view = B.headless_view(W, H)
    plugins = [B.GaussianSplattingPlugin(0) for _ in range(CTX)]
    handles = [p.add_cloud(cloud) for p in plugins]
    res = {"card": card(), "n": N, "width": W, "height": H, "global_scale": SCALE, "frames": a.frames, "times": {}}
    for t in TIMES:
        s = B.CloudSettings(gaussian_mode=B.GaussianMode.Gaussian4d, global_scale=SCALE, time=t)
        p0, h0 = plugins[0], handles[0]
        for _ in range(5):
            p0.render_view(h0, s, view, to_host=False)
        rec, _ = p0.projected()
        bb = rec[:, 6:8].view(np.uint32)
        drawn = int((((bb[:, 0] & 0xFFFF) <= (bb[:, 0] >> 16)) & ((bb[:, 1] & 0xFFFF) <= (bb[:, 1] >> 16))).sum())
        stage = p0.stage_times_us().tolist()
        t0 = time.perf_counter()
        for _ in range(a.frames):
            p0.render_view(h0, s, view, to_host=False)
        one = (time.perf_counter() - t0) * 1e3 / a.frames
        for p, h in zip(plugins, handles):   # warm the queued path
            p.render_view(h, s, view, to_host=False, asynchronous=True)
        for p in plugins:
            p.sync()
        t0 = time.perf_counter()
        for k in range(a.frames):
            plugins[k % CTX].render_view(handles[k % CTX], s, view, to_host=False, asynchronous=True)
        for p in plugins:
            p.sync()
        flight = (time.perf_counter() - t0) * 1e3 / a.frames
        res["times"][str(t)] = {"drawn_fraction": drawn / N, "n_visible": int(len(rec)), "ms_per_frame_sync": one,
                                "ms_per_frame_3_in_flight": flight, "projection_us": stage[2], "stage_us": stage}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    for p in plugins:
        p.destroy()


if __name__ == "__main__":
    main()
